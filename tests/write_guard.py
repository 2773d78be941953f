"""Guard-banded output buffers: what a kernel writes, and where.

An output or accumulator is handed to a kernel as a view into a larger buffer: a front guard of whole rows, a row pitch ``ld`` wider than
the region (so every row is followed by a ``[width, ld)`` gap) and a back guard.  The whole buffer starts as a sentinel bit pattern -- a NaN
with a recognisable payload for fp32 / bf16, a fixed pattern for fp64 and the integer types -- so that a store or atomic that lands outside
the region changes bits the test owns and can read back, instead of corrupting the allocator's slack (or, inside the engine's packed
gradient and statistics buffers, the neighbouring parameter's gradient).

    g = Guarded((rows, width), torch.bfloat16, ld=width + 8)    # g.view is the [rows, width] region, g.ld its pitch
    kernel(..., g.ptr, g.ld)
    g.check_bands()                                              # guards and gaps bit-identical to the sentinel
    g.check_written()                                            # no sentinel survives inside the region

Accumulated outputs: ``g.fill(P)`` puts a prior into the region, the test then compares the region with ``P + out0``.

Used by test_write_contract_gpu.py on device buffers; test_write_contract_cpu.py runs the negative controls on CPU tensors."""
import torch

# sentinel bit patterns, per element size: quiet NaNs with a payload (fp32 0x7fc5a5a5, bf16 0x7fa5, fp64 0x7ff8a5a5a5a5a5a5) -- a kernel that
# reads one back propagates a NaN -- and the same pattern for the integer types of the same width
_SENTINEL_BITS = {1: 0xA5, 2: 0x7FA5, 4: 0x7FC5A5A5, 8: 0x7FF8A5A5A5A5A5A5}
_INT_OF_SIZE = {1: torch.int8, 2: torch.int16, 4: torch.int32, 8: torch.int64}


def _signed(bits, size):
    return bits - (1 << (8 * size)) if bits >= 1 << (8 * size - 1) else bits


def sentinel_bits(dtype):
    size = torch.empty((), dtype=dtype).element_size()
    return _signed(_SENTINEL_BITS[size], size)


def bits(t):
    """the raw bit pattern of a tensor as the signed integer type of its element size"""
    return t.view(_INT_OF_SIZE[t.element_size()])


class Guarded:
    """A [rows, width] region (``shape`` = (rows, width), or (n,) for a vector) at pitch ``ld`` inside a sentinel-filled buffer with
    ``guard_rows`` whole rows in front and behind (at least ``min_guard`` elements each).  The front guard is rounded up to 128 bytes so
    the region keeps the alignment the kernels require of their operands."""

    def __init__(self, shape, dtype, device="cuda", ld=None, guard_rows=128, min_guard=1024):
        self.vector = len(shape) == 1
        self.rows, self.width = (1, int(shape[0])) if self.vector else (int(shape[0]), int(shape[1]))
        self.ld = int(ld) if ld is not None else self.width
        assert self.ld >= self.width
        esz = torch.empty((), dtype=dtype).element_size()
        front = max(guard_rows * self.ld, min_guard)
        front = -(-front * esz // 128) * 128 // esz
        back = max(guard_rows * self.ld, min_guard)
        self.front, self.back = front, back
        n = front + self.rows * self.ld + back
        self.dtype = dtype
        self.buf = torch.empty(n, dtype=dtype, device=device)
        self.sentinel = sentinel_bits(dtype)
        bits(self.buf).fill_(self.sentinel)
        self.padded = self.buf[front:front + self.rows * self.ld].view(self.rows, self.ld)
        self.view = self.padded[:, :self.width]

    @property
    def ptr(self):
        return self.view.data_ptr()

    def fill(self, values):
        """put a prior (an accumulator's previous contents) into the region; the guards and gaps keep the sentinel"""
        self.view.copy_(torch.as_tensor(values).to(self.view.device, self.dtype).reshape(self.view.shape))
        return self

    def region(self):
        """the region as a contiguous tensor (rows x width, or the vector)"""
        return self.view.clone().reshape(-1) if self.vector else self.view.clone()

    def _outside(self):
        b = bits(self.buf)
        return [("front guard", b[:self.front]), ("back guard", b[self.front + self.rows * self.ld:]),
                ("row gap", bits(self.padded[:, self.width:]).reshape(-1))]

    def check_bands(self, what=""):
        """every guard element and every element of the [width, ld) row gaps still holds the sentinel, bit for bit"""
        for name, part in self._outside():
            bad = part != self.sentinel
            if bool(bad.any()):
                idx = [int(i) for i in bad.nonzero().reshape(-1)[:4]]
                raise AssertionError(f"{what}: {int(bad.sum())} element(s) of the {name} overwritten (first at {idx}; "
                                     f"region {self.rows} x {self.width}, ld {self.ld})")

    def check_written(self, what="", cols=None):
        """no element of the region (or of its columns ``cols``, a slice) still holds the sentinel: the kernel wrote every one.  For floating
        types every element must also be finite: a kernel that adds into a "written" output instead of storing turns the NaN sentinel into
        another NaN (the device's canonical one), which the bit comparison alone would take for a write."""
        v = self.view if cols is None else self.view[:, cols]
        left = bits(v.contiguous()) == self.sentinel
        if bool(left.any()):
            idx = [tuple(int(j) for j in i) for i in left.nonzero()[:4]]
            raise AssertionError(f"{what}: {int(left.sum())}/{left.numel()} region element(s) never written (first at {idx})")
        if self.dtype.is_floating_point:
            bad = ~torch.isfinite(v.float())
            if bool(bad.any()):
                idx = [tuple(int(j) for j in i) for i in bad.nonzero()[:4]]
                raise AssertionError(f"{what}: {int(bad.sum())}/{bad.numel()} region element(s) not finite (first at {idx}): "
                                     "a NaN prior added into instead of overwritten?")

    def check_untouched(self, what="", cols=None):
        """the region's columns ``cols`` (a slice) still hold the sentinel: outputs documented to touch only some columns"""
        v = self.view if cols is None else self.view[:, cols]
        bad = bits(v.contiguous()) != self.sentinel
        if bool(bad.any()):
            raise AssertionError(f"{what}: {int(bad.sum())} element(s) written in columns the kernel must leave alone")

    def check(self, what=""):
        self.check_bands(what)
        self.check_written(what)
        return self.region()
