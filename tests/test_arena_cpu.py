"""workspace.Arena on CPU tensors: scratch sized from the record of what earlier calls carved, carves that do not fit get tensors of their
own and raise the record, and the fp64 -> fp32 conversion covers both kinds of carve."""
import pytest
import torch

from ml_cvnets_b200.workspace import Arena


@pytest.fixture
def own_carves(monkeypatch):
    """Counts the carves that got a tensor of their own instead of a slice of the arena's buffers."""
    calls = []
    own = Arena._own

    def counting(n, like):
        calls.append((n, like.dtype))
        return own(n, like)

    monkeypatch.setattr(Arena, "_own", staticmethod(counting))
    return calls


def _carve(ar, big=1):
    """The same carve sequence as a module backward: fp32 and fp64 interleaved, sizes that need rounding."""
    return [ar.f32(3, 5), ar.f64(2, 3), ar.f32(7 * big), ar.f64(5 * big)]


def _spans(views):
    return sorted((v.data_ptr(), v.data_ptr() + v.numel() * v.element_size()) for v in views)


def _check_carves(views, shapes):
    assert [tuple(v.shape) for v in views] == shapes
    for v in views:
        assert v.data_ptr() % 16 == 0
        assert not v.any()
    spans = _spans(views)
    assert all(hi <= lo for (_, hi), (lo, _) in zip(spans, spans[1:])), spans


def test_first_call_carves_its_own_tensors_and_records_totals(own_carves):
    rec = [0, 0]
    views = _carve(Arena(rec, "cpu"))
    _check_carves(views, [(3, 5), (2, 3), (7,), (5,)])
    assert len(own_carves) == 4
    assert rec == [16 + 8, 6 + 6]  # fp32 carves rounded to 4 floats, fp64 carves to 2 doubles


def test_second_call_uses_one_buffer_per_dtype(own_carves):
    rec = [0, 0]
    first = _carve(Arena(rec, "cpu"))
    for v in first:
        v.fill_(1.0)  # the next call must still see zeros
    own_carves.clear()
    ar = Arena(rec, "cpu")
    views = _carve(ar)
    assert own_carves == []
    assert ar.b32.numel() == 24 and ar.b64.numel() == 12
    _check_carves(views, [tuple(v.shape) for v in first])
    for v in views:
        buf = ar.b32 if v.dtype == torch.float32 else ar.b64
        assert v.untyped_storage().data_ptr() == buf.untyped_storage().data_ptr()
    assert rec == [24, 12]


def test_larger_call_overflows_and_raises_the_record(own_carves):
    rec = [24, 12]
    ar = Arena(rec, "cpu")
    views = _carve(ar, big=3) + [ar.f32(1)]
    _check_carves(views, [(3, 5), (2, 3), (21,), (15,), (1,)])
    in_buf = [v.untyped_storage().data_ptr() in (ar.b32.untyped_storage().data_ptr(), ar.b64.untyped_storage().data_ptr()) for v in views]
    assert in_buf == [True, True, False, False, False]  # a carve past the buffer's end, and every carve after it, is a tensor of its own
    assert own_carves == [(24, torch.float32), (16, torch.float64), (4, torch.float32)]
    assert rec == [16 + 24 + 4, 6 + 16]
    own_carves.clear()
    _check_carves(_carve(Arena(rec, "cpu"), big=3), [(3, 5), (2, 3), (21,), (15,)])
    assert own_carves == []


def test_cast_covers_buffer_and_own_carves(own_carves):
    rec = [0, 8]
    ar = Arena(rec, "cpu")
    a, b, c = ar.f64(2, 3), ar.f64(7), ar.f64(2, 4)
    assert len(own_carves) == 2  # b and c do not fit
    g = torch.Generator().manual_seed(3)
    for v in (a, b, c):
        v.copy_(torch.randn(v.shape, generator=g, dtype=torch.float64) * 1e3)
    ar.cast()
    for v in (a, a[1], b, c, c[0], c[1]):  # rows: the way a backward hands over (sum, sum of squares) pairs
        out = ar.as_f32(v)
        assert out.dtype == torch.float32 and out.shape == v.shape
        assert torch.equal(out, v.float())
