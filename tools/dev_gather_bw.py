"""Development: the bandwidth one GPU sustains on random 208-byte and 128-byte segment gathers with the launch shape of the
K1-D upper pass (tools/dev_gather_bw.cu) -- the denominator for that pass's from-shapes traffic in DESIGN.md 3a.
    python tools/dev_gather_bw.py
Builds the stand-alone program with nvcc into a temporary directory, prints the card's name, power limit and maximum SM
clock, then one JSON line per segment size."""
import os, subprocess, sys, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from recsys2019_deeplearning_evaluation_b200 import build as B

src = os.path.join(ROOT, "tools", "dev_gather_bw.cu")
with tempfile.TemporaryDirectory() as tmp:
    exe = os.path.join(tmp, "dev_gather_bw")
    subprocess.check_call([B._nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-o", exe, src])
    subprocess.call(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"])
    sys.exit(subprocess.call([exe]))
