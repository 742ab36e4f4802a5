"""Build a VARIANT of the library for same-box A/B runs: csrc/<file>.cu recompiled with extra -D flags, linked with the product's
other objects into tools/_trace/libbagel_b200_<name>.so (git-ignored, travels to the GPU box). A tool then loads it by setting
PERF_LIB=<path> (tools/gpu_perf_attn.py) — the package itself only ever loads bagel_b200/libbagel_b200.so.
  python tools/build_variant.py stages4 attn -DBAGEL_ATTN_STAGES128=4"""
import subprocess, sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from bagel_b200 import build as bb

name, stem, flags = sys.argv[1], sys.argv[2], sys.argv[3:]
bb.build()
out_dir = ROOT / "tools" / "_trace"
out_dir.mkdir(parents=True, exist_ok=True)
obj = out_dir / f"{stem}_{name}.o"
subprocess.check_call([bb._nvcc(), *bb.NVCC_FLAGS, *flags, "-c", str(bb.CSRC / f"{stem}.cu"), "-o", str(obj)])
objs = [str(o) for o in sorted((bb.PKG_DIR / "build").glob("*.o")) if o.name != f"{stem}.o"] + [str(obj)]
lib = out_dir / f"libbagel_b200_{name}.so"
subprocess.check_call([bb._nvcc(), "-shared", "-o", str(lib), *objs, "-gencode", "arch=compute_90a,code=sm_90a", "-lcuda"])
print("built", lib)
