"""Development timing of DIVERSITY_SIMILARITY in EvaluatorHoldout on one GPU:
    python tools/dev_diversity_bench.py [--out FILE.json] [--shapes ml1m,20k] [--rounds R] [--oracle-users-1024 N]
Shapes: ML-1M (6 040 x 3 706) with the diversity matrix D in fp32 and in fp64, and a 20 000 x 20 000 catalogue with an
fp32 D (1.6 GB, far beyond the 50 MB L2).  D is uniform random in [0, 1] (the kernel's reads do not depend on the values).
The model is MF-BPR with 64 seeded random factors (scoring cost does not depend on how the factors were trained).
Cutoffs [5, 10, 20, 50, 100] and [1024].  For each case, alternating `--rounds` times: a whole `evaluateRecommender` call
without and with the diversity object (host clock around calls that end in a device synchronise), so the difference is
the added cost per evaluation; the two metric dicts are compared on every shared key (max relative difference: the fp64
atomics across users may add in another order).  On ML-1M the oracle's per-user transcription of the reference's loop
(`oracle.diversity_oracle.diversity_similarity`, float64) is timed on the same lists: all users for the short cutoffs,
the first `--oracle-users-1024` users for cutoff 1 024, whose per-user time is scaled to all users and marked as such.
The card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from oracle.diversity_oracle import diversity_similarity
from recsys2019_deeplearning_evaluation_b200 import recommenders as R
from recsys2019_deeplearning_evaluation_b200.evaluation import Diversity_similarity, EvaluatorHoldout
from recsys2019_deeplearning_evaluation_b200.synth import synth_urm

SHAPES = {"ml1m": (6040, 3706, 0.045, ("float32", "float64")), "20k": (20000, 20000, 0.005, ("float32",))}
CUTOFF_SETS = ([5, 10, 20, 50, 100], [1024])


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name()


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def max_rel_diff_shared(a, b):
    d = 0.0
    for c in b:
        for k in b[c]:
            x, y = a[c][k], b[c][k]
            if np.isnan(x) and np.isnan(y):
                continue
            d = max(d, abs(x - y) / max(abs(y), 1e-300))
    return d


def oracle_seconds(D, lists, cutoffs):
    D64 = np.asarray(D, dtype=np.float64)
    t0 = time.perf_counter()
    for r in lists:
        for c in cutoffs:
            diversity_similarity(D64, r[:c])
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--shapes", default="ml1m,20k")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--oracle-users-1024", type=int, default=300)
    args = ap.parse_args()
    report = {"card": card(), "shapes": {}}
    print(report["card"], flush=True)
    for name in args.shapes.split(","):
        n_users, n_items, density, dtypes = SHAPES[name]
        train = synth_urm(n_users, n_items, density, seed=1, popularity=0.8)
        test = synth_urm(n_users, n_items, 0.002 if n_items < 10000 else 0.0005, seed=2)
        rng = np.random.default_rng(3)
        rec = R.MatrixFactorization_BPR_Cython(train, verbose=False)
        rec.USER_factors = (rng.standard_normal((n_users, 64)) * 0.1).astype(np.float32)
        rec.ITEM_factors = (rng.standard_normal((n_items, 64)) * 0.1).astype(np.float32)
        shape = {"n_users": n_users, "n_items": n_items, "train_nnz": int(train.nnz), "cases": {}}
        for dtype in dtypes:
            D = rng.random((n_items, n_items), dtype=np.float32 if dtype == "float32" else np.float64)
            div = Diversity_similarity(D)
            for cutoffs in CUTOFF_SETS:
                ev_plain = EvaluatorHoldout(test, cutoffs, verbose=False)
                ev_div = EvaluatorHoldout(test, cutoffs, diversity_object=div, verbose=False)
                ev_plain.evaluateRecommender(rec)  # warm-up: module loads, caches, the upload of D
                ev_div.evaluateRecommender(rec)
                r = {"n_eval": len(ev_div.users_to_evaluate), "plain_s": [], "diversity_s": [], "max_rel_diff_shared_keys": []}
                for _ in range(args.rounds):
                    t, res_plain = wall(lambda: ev_plain.evaluateRecommender(rec))
                    r["plain_s"].append(t)
                    t, res_div = wall(lambda: ev_div.evaluateRecommender(rec))
                    r["diversity_s"].append(t)
                    r["max_rel_diff_shared_keys"].append(max_rel_diff_shared(res_div[0], res_plain[0]))
                r["added_s_median"] = float(np.median(r["diversity_s"]) - np.median(r["plain_s"]))
                r["DIVERSITY_SIMILARITY"] = {c: res_div[0][c]["DIVERSITY_SIMILARITY"] for c in cutoffs}
                if name == "ml1m":
                    users = np.asarray(ev_div.users_to_evaluate)
                    n_or = len(users) if max(cutoffs) <= 100 else min(args.oracle_users_1024, len(users))
                    lists = [np.asarray(x, dtype=np.int64) for x in rec.recommend(users[:n_or], cutoff=max(cutoffs))]
                    t = oracle_seconds(D, lists, cutoffs)
                    r["oracle_users_timed"] = n_or
                    r["oracle_s"] = t
                    r["oracle_s_all_users" + ("" if n_or == len(users) else "_scaled")] = t * len(users) / n_or
                key = "%s_cut%s" % (dtype, "-".join(map(str, cutoffs)))
                shape["cases"][key] = r
                print(name, key, json.dumps(r), flush=True)
                del ev_plain, ev_div
            del div, D
            torch.cuda.empty_cache()
        report["shapes"][name] = shape
    txt = json.dumps(report, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(txt)
    print(txt)


if __name__ == "__main__":
    main()
