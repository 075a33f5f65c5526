"""Development: build a variant of libb200rec.so with extra -D flags for A/B timing on the GPU box.

usage: python tools/build_variant.py NAME -DB200_SELT=256 ...   ->  recsys2019_deeplearning_evaluation_b200/_variants/libb200rec_NAME.so
Select it at run time with B200REC_LIB=<path>."""
import glob, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from recsys2019_deeplearning_evaluation_b200 import build as B

name, defs = sys.argv[1], sys.argv[2:]
out_dir = os.path.join(B.PKG, "_variants")
obj_dir = os.path.join(out_dir, "obj_" + name)
os.makedirs(obj_dir, exist_ok=True)
objs = []
for src in sorted(glob.glob(os.path.join(B.CSRC, "*.cu"))):
    base = os.path.basename(src)[:-3]
    if base == "sim_topk":
        obj = os.path.join(obj_dir, base + ".o")
        subprocess.check_call([B._nvcc()] + B.NVCC_FLAGS + defs + ["-c", src, "-o", obj])
    else:
        obj = os.path.join(B.OBJ, base + ".o")
    objs.append(obj)
lib = os.path.join(out_dir, "libb200rec_%s.so" % name)
subprocess.check_call([B._nvcc(), "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", lib] + objs)
print(lib)
