"""Static check (no GPU): every name a function of bagel_b200 / bench.py / __graft_entry__.py reads is bound somewhere
(argument, local, enclosing scope, module global or builtin). The GPU-only code paths cannot be executed in the build
container, so a typo there would otherwise first show up on the GPU machine."""
import ast
import builtins
import glob
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bound_names(node):
    names = set()
    for n in ast.walk(node):
        if isinstance(n, ast.Name) and isinstance(n.ctx, (ast.Store, ast.Del)):
            names.add(n.id)
        elif isinstance(n, (ast.FunctionDef, ast.AsyncFunctionDef, ast.ClassDef)):
            names.add(n.name)
        elif isinstance(n, ast.arg):
            names.add(n.arg)
        elif isinstance(n, (ast.Import, ast.ImportFrom)):
            for a in n.names:
                names.add((a.asname or a.name).split(".")[0])
        elif isinstance(n, ast.ExceptHandler) and n.name:
            names.add(n.name)
    return names


def _check(path):
    tree = ast.parse(open(path).read())
    module_names = _bound_names(tree) | set(dir(builtins)) | {"__file__", "__name__"}
    problems = []

    def visit(fn, outer):
        scope = outer | _bound_names(fn)
        for n in ast.walk(fn):
            if isinstance(n, ast.Name) and isinstance(n.ctx, ast.Load) and n.id not in scope:
                problems.append(f"{os.path.relpath(path, ROOT)}:{n.lineno}: undefined name {n.id!r} in {fn.name}()")

    for node in ast.walk(tree):
        if isinstance(node, (ast.FunctionDef, ast.AsyncFunctionDef)):
            visit(node, module_names)
    return problems


def test_no_undefined_names():
    files = glob.glob(os.path.join(ROOT, "bagel_b200", "*.py")) + [os.path.join(ROOT, "bench.py"),
                                                                   os.path.join(ROOT, "__graft_entry__.py")]
    files += glob.glob(os.path.join(ROOT, "tools", "*.py"))
    problems = [p for f in sorted(files) for p in _check(f)]
    assert not problems, "\n".join(problems)


def test_attention_exp2_polynomial_constants():
    """The FMA-pipe exp2 of csrc/attn.cu (ex2_poly2): fp32 emulation of the magic-number split + degree-3 polynomial + exponent
    add, with the constants parsed from the source; relative error against 2^x over the range the kernel can produce."""
    import re
    import numpy as np
    src = open(os.path.join(ROOT, "bagel_b200", "csrc", "attn.cu")).read()
    body = src[src.index("ex2_poly2(float2 x)"):]
    body = body[:body.index("return r;")]
    c1, c2, c3 = (np.float32(float(re.search(rf"c{k} = make_float2\(([0-9.]+)f", body).group(1))) for k in (1, 2, 3))
    magic = np.float32(float(re.search(r"magic = make_float2\(([0-9.]+)f", body).group(1)))
    assert magic == np.float32(12582912.0)
    x = np.concatenate([np.linspace(-126.0, 60.0, 400001), np.array([-1e30, -126.5, -0.5, 0.0, 0.49999, 0.5, 0.50001])]).astype(np.float32)
    x = np.maximum(x, np.float32(-126.0))
    t = (x + magic).astype(np.float32)
    n = (t - magic).astype(np.float32)
    f = (x - n).astype(np.float32)
    assert np.all(np.abs(f) <= 0.5)
    q = (f * c3 + c2).astype(np.float32)
    q = (q * f + c1).astype(np.float32)
    q = (q * f + np.float32(1.0)).astype(np.float32)
    bits = (q.view(np.int32).astype(np.int64) + ((t.view(np.int32).astype(np.int64) << 23) & 0xFFFFFFFF)) & 0xFFFFFFFF
    r = bits.astype(np.uint32).view(np.float32).astype(np.float64)
    ref = np.exp2(x.astype(np.float64))
    ok = ref > 1e-37                      # 2^-126 itself lands on the denormal boundary
    rel = np.abs(r[ok] - ref[ok]) / ref[ok]
    assert rel.max() < 1.2e-4, rel.max()
