"""A/B variants of the library for kernel tuning: tools/build_variants.py NAME=-DFLAG[,-DFLAG...] ...
Objects of the unchanged translation units are compiled once; only frontend_kernels.cu is rebuilt per variant.
Output: build_variants/librgbdslam_b200.NAME.so (git-ignored, travels to the GPU box)."""
import subprocess, sys, shutil
from pathlib import Path
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from rgbdslam_v2_b200.build import CSRC, _nvcc, sources
OUT = ROOT / "build_variants"; OBJ = OUT / "obj"; OBJ.mkdir(parents=True, exist_ok=True)
FL = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-ccbin", shutil.which("g++")]
TUNED = {"frontend_kernels.cu", "hamming_tc.cu", "posegraph.cu"}
def cc(src, obj, extra=()):
    subprocess.run([_nvcc(), *FL, *extra, "-c", str(src), "-o", str(obj)], check=True)
common = []
for s in sources():
    if s.name in TUNED: continue
    o = OBJ / (s.stem + ".o")
    if not o.exists() or o.stat().st_mtime < max(p.stat().st_mtime for p in [s, *CSRC.glob("*.h"), *CSRC.glob("*.cuh")]): cc(s, o)
    common.append(o)
for spec in sys.argv[1:]:
    name, _, flags = spec.partition("=")
    extra = [f for f in flags.split(",") if f]
    objs = []
    for t in sorted(TUNED):
        o = OBJ / f"{Path(t).stem}.{name}.o"; cc(CSRC / t, o, extra); objs.append(o)
    lib = OUT / f"librgbdslam_b200.{name}.so"
    subprocess.run([_nvcc(), "-shared", "-ldl", "-gencode", "arch=compute_90a,code=sm_90a", "-o", str(lib), *map(str, common + objs), "-ccbin", shutil.which("g++")], check=True)
    print("built", lib)
