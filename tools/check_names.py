"""Poor man's pyflakes (none is installed and there is no network): report names that are loaded but never bound anywhere in the module
and are not builtins.  Run before every GPU submission -- a NameError in a GPU-only code path costs a GPU call.

    python tools/check_names.py ml-cvnets_b200/*.py bench.py tests/*.py
"""
import ast
import builtins
import sys


def check(path):
    tree = ast.parse(open(path).read(), path)
    bound = set(dir(builtins)) | {"__file__", "__name__", "__doc__"}
    for node in ast.walk(tree):
        if isinstance(node, (ast.Import, ast.ImportFrom)):
            for a in node.names:
                bound.add((a.asname or a.name).split(".")[0])
        elif isinstance(node, (ast.FunctionDef, ast.AsyncFunctionDef, ast.ClassDef)):
            bound.add(node.name)
            if not isinstance(node, ast.ClassDef):
                for a in node.args.args + node.args.kwonlyargs + node.args.posonlyargs:
                    bound.add(a.arg)
                if node.args.vararg:
                    bound.add(node.args.vararg.arg)
                if node.args.kwarg:
                    bound.add(node.args.kwarg.arg)
        elif isinstance(node, ast.Lambda):
            for a in node.args.args + node.args.kwonlyargs + node.args.posonlyargs + [node.args.vararg, node.args.kwarg]:
                if a is not None:
                    bound.add(a.arg)
        elif isinstance(node, ast.Name) and isinstance(node.ctx, (ast.Store, ast.Del)):
            bound.add(node.id)
        elif isinstance(node, ast.ExceptHandler) and node.name:
            bound.add(node.name)
        elif isinstance(node, ast.comprehension):
            for n in ast.walk(node.target):
                if isinstance(n, ast.Name):
                    bound.add(n.id)
        elif isinstance(node, (ast.Global, ast.Nonlocal)):
            bound.update(node.names)
    bad = []
    for node in ast.walk(tree):
        if isinstance(node, ast.Name) and isinstance(node.ctx, ast.Load) and node.id not in bound:
            bad.append((node.lineno, node.id))
    return bad


if __name__ == "__main__":
    rc = 0
    for p in sys.argv[1:]:
        for ln, name in check(p):
            print(f"{p}:{ln}: undefined name '{name}'")
            rc = 1
    sys.exit(rc)
