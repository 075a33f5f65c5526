"""Build recipe for oracle/_ref: the reference's OWN Cython hot loops, compiled unmodified.

TEST INFRASTRUCTURE ONLY (see oracle/README.md).  Nothing under recsys2019_deeplearning_evaluation_b200/
may import this.

The three extension modules are compiled from the sources where they lie under /root/reference
(read-only) -- no reference source is copied into this repository.  Only the resulting `.so` files are
kept, in oracle/_ref/ (git-ignored):

  Base/Similarity/Cython/Compute_Similarity_Cython.pyx                    -> Compute_Similarity_Cython*.so
  SLIM_BPR/Cython/SLIM_BPR_Cython_Epoch.pyx                               -> SLIM_BPR_Cython_Epoch*.so
  MatrixFactorization/Cython/MatrixFactorization_Cython_Epoch.pyx         -> MatrixFactorization_Cython_Epoch*.so

Flags follow the reference's own build (CythonCompiler/compile_script.py:40-44: `-O2`, numpy include).
SLIM_BPR needs Cython-3 `legacy_implicit_noexcept` (its qsort comparators, pyx:991,995, predate the
Cython 3 exception-spec change); the source itself is not edited.

Usage:  python oracle/build_ref.py [--force]
"""
import glob
import os
import shutil
import subprocess
import sys
import tempfile

REF = os.environ.get("B200REC_REFERENCE", "/root/reference")
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")

MODULES = [
    ("Compute_Similarity_Cython", "Base/Similarity/Cython/Compute_Similarity_Cython.pyx"),
    ("SLIM_BPR_Cython_Epoch", "SLIM_BPR/Cython/SLIM_BPR_Cython_Epoch.pyx"),
    ("MatrixFactorization_Cython_Epoch", "MatrixFactorization/Cython/MatrixFactorization_Cython_Epoch.pyx"),
]

_SETUP = r'''
import sys, numpy
from setuptools import setup, Extension
from Cython.Build import cythonize
name, src, build_dir = sys.argv[1], sys.argv[2], sys.argv[3]
del sys.argv[1:4]
ext = Extension(name, [src], extra_compile_args=["-O2"], include_dirs=[numpy.get_include()])
setup(name=name, ext_modules=cythonize([ext], build_dir=build_dir,
      compiler_directives={"legacy_implicit_noexcept": True, "language_level": 3}))
'''


def have(name):
    return bool(glob.glob(os.path.join(OUT, name + "*.so")))


def build_one(name, rel, force=False):
    if have(name) and not force:
        return True
    src = os.path.join(REF, rel)
    if not os.path.exists(src):
        return False
    os.makedirs(OUT, exist_ok=True)
    with tempfile.TemporaryDirectory(prefix="b200rec_ref_") as tmp:
        script = os.path.join(tmp, "setup_one.py")
        with open(script, "w") as f:
            f.write(_SETUP)
        # cwd = tmp so that neither the generated .c nor build/ lands in the repo or in /root/reference
        cmd = [sys.executable, script, name, src, os.path.join(tmp, "cy"),
               "build_ext", "--build-lib", tmp, "--build-temp", os.path.join(tmp, "obj")]
        r = subprocess.run(cmd, cwd=tmp, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout[-4000:])
            raise RuntimeError("reference module %s failed to compile" % name)
        for so in glob.glob(os.path.join(tmp, name + "*.so")):
            shutil.copy2(so, OUT)
    return have(name)


def build_all(force=False):
    """Returns {module: bool}.  No-op (False entries) when /root/reference is absent and nothing is prebuilt."""
    return {name: build_one(name, rel, force) for name, rel in MODULES}


if __name__ == "__main__":
    res = build_all(force="--force" in sys.argv)
    print(res)
    sys.exit(0 if all(res.values()) else 1)
