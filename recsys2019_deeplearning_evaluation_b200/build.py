"""In-tree build of libb200rec.so (sm_90a only).  `python -m recsys2019_deeplearning_evaluation_b200.build`.
(The checkers -- the C oracle and the compiled reference -- are built by oracle/build_oracle.py and oracle/build_ref.py,
called from __graft_entry__.build().)

nvcc cross-compiles without a GPU.  The resulting .so and objects are git-ignored.  Incremental: a source is recompiled only when it (or a header) is newer than its object.
"""
import glob
import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
OBJ = os.path.join(PKG, "csrc", "_obj")
LIB = os.path.join(PKG, "libb200rec.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-I", os.path.join(ROOT, "include"), "-I", CSRC,
    "--expt-relaxed-constexpr", "-Xptxas", "-v",
]


def _nvcc():
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found; libb200rec.so cannot be built (there is no CPU fallback)")


def _newer(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build_lib(force=False, verbose=False):
    nvcc = _nvcc()
    os.makedirs(OBJ, exist_ok=True)
    headers = glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(ROOT, "include", "*.h"))
    sources = sorted(glob.glob(os.path.join(CSRC, "*.cu")))
    objs, rebuilt, logs = [], False, {}
    for src in sources:
        obj = os.path.join(OBJ, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        if force or _newer(obj, [src] + headers):
            cmd = [nvcc] + NVCC_FLAGS + ["-c", src, "-o", obj]
            r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
            logs[os.path.basename(src)] = r.stdout
            if r.returncode != 0:
                sys.stderr.write(r.stdout)
                raise RuntimeError("nvcc failed on %s" % src)
            if verbose:
                sys.stderr.write(r.stdout)
            rebuilt = True
    if rebuilt or force or _newer(LIB, objs):
        cmd = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB] + objs
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout)
            raise RuntimeError("link of libb200rec.so failed")
    with open(os.path.join(OBJ, "ptxas.log"), "a" if not force else "w") as f:
        for k, v in logs.items():
            f.write("==== %s\n%s\n" % (k, v))
    return LIB


if __name__ == "__main__":
    print(build_lib(force="--force" in sys.argv, verbose="-v" in sys.argv))
