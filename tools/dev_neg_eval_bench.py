"""Development timing of EvaluatorNegativeItemSample on one GPU:
    python tools/dev_neg_eval_bench.py [--out FILE.json] [--shapes ml1m,pinterest,c5] [--old-users N] [--rounds R]
Leave-one-out + 100-negative shapes (one test item and 100 sampled negatives per user): ML-1M (6 040 x 3 706), Pinterest-like
(55 187 x 9 916) and C5-like (1 M x 200 K; 20 train items per user).  Models: ItemKNN (fitted), MF-BPR (64 factors) and IALS
(128 factors) with seeded random factors (scoring cost does not depend on how the factors were trained), EASE_R with topK=None
(fitted; not at C5-like, where its dense 200 K^2 B does not fit).  For each model, alternating `--rounds` times:
  * new: evaluateRecommender on all users (blocks of users, candidate kernels), users/s over the whole call;
  * old: the one-user-per-step path this evaluator used before (full-catalogue score row, candidate mask, seen mask, top-N
    over all items, accumulate), on the first `--old-users` evaluated users, users/s; the new path is run on the same
    users too and its metric dict compared with the old one (max relative difference over all metrics and cutoffs);
  * fallback: the scoring step alone over all blocks, family kernel (_candidate_scores_device) against block + gather
    (_candidate_scores_by_block), device time.
The card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import scipy.sparse as sps
import torch

from recsys2019_deeplearning_evaluation_b200 import recommenders as R
from recsys2019_deeplearning_evaluation_b200.evaluation import EvaluatorNegativeItemSample
from recsys2019_deeplearning_evaluation_b200.synth import synth_urm

SHAPES = {"ml1m": (6040, 3706, 0.045), "pinterest": (55187, 9916, 0.0027), "c5": (1000000, 200000, 0.0001)}


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name()


def loo_data(n_users, n_items, density, seed):
    """train, test (one item per user), 100 sampled negatives per user (duplicates merged)."""
    rng = np.random.default_rng(seed)
    train = synth_urm(n_users, n_items, density, seed=seed, popularity=0.8)
    rows = np.arange(n_users)
    test = sps.csr_matrix((np.ones(n_users, np.float32), (rows, rng.integers(0, n_items, n_users))), shape=(n_users, n_items))
    neg_cols = rng.integers(0, n_items, (n_users, 100)).ravel()
    neg = sps.csr_matrix((np.ones(len(neg_cols), np.float32), (np.repeat(rows, 100), neg_cols)), shape=(n_users, n_items))
    return train, test, neg


class OldPathEvaluator(EvaluatorNegativeItemSample):
    """The previous one-user-per-step loop, kept here only as the timing / result baseline."""

    def _evaluate_blocks(self, rec, users, block_size, st):
        cutoff = int(min(self.max_cutoff, self.n_items))
        for u in users:
            d_users = rec._users_tensor(np.atleast_1d(u))
            scores = rec._masked_scores_device(d_users, remove_seen_flag=self.exclude_seen,
                                               items_to_compute=self._get_user_specific_items_to_compute(int(u)),
                                               remove_custom_items_flag=self.ignore_items_flag)
            items, vals = rec._topn_device(scores, cutoff)
            self._accumulate(st, d_users, items, vals, cutoff)


def models(name, train, seed):
    n_users, n_items = train.shape
    rng = np.random.default_rng(seed)
    out = []
    knn = R.ItemKNNCFRecommender(train, verbose=False)
    knn.fit(topK=100, shrink=10)
    out.append(("ItemKNN", knn))
    for label, cls, f in (("MF-BPR", R.MatrixFactorization_BPR_Cython, 64), ("IALS", R.IALSRecommender, 128)):
        m = cls(train, verbose=False)
        m.USER_factors = (rng.standard_normal((n_users, f)) * 0.1).astype(np.float32)
        m.ITEM_factors = (rng.standard_normal((n_items, f)) * 0.1).astype(np.float32)
        out.append((label, m))
    if name != "c5":
        ease = R.EASE_R_Recommender(train, verbose=False)
        ease.fit(topK=None, l2_norm=100.0, verbose=False)
        out.append(("EASE_R", ease))
    return out


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def max_rel_diff(a, b):
    d = 0.0
    for c in a:
        for k in a[c]:
            x, y = a[c][k], b[c][k]
            if np.isnan(x) and np.isnan(y):
                continue
            d = max(d, abs(x - y) / max(abs(y), 1e-300))
    return d


def scoring_time(ev, rec, block_size, by_block):
    """Device time of the scoring step alone over all blocks of the evaluator's users."""
    n = len(ev.users_to_evaluate)
    d_users, d_ptr, d_idx = ev._cand_device(torch.device("cuda", torch.cuda.current_device()))
    starts = list(range(0, n, block_size))
    longest = max(int(ev._cand_ptr[min(s + block_size, n)] - ev._cand_ptr[s]) for s in starts)
    out = torch.empty(max(longest, 1), dtype=torch.float32, device="cuda")
    fn = rec._candidate_scores_by_block if by_block else rec._candidate_scores_device
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for s in starts:
        nb = min(block_size, n - s)
        fn(d_users[s:s + nb], d_ptr[s:s + nb + 1], d_idx, out)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--shapes", default="ml1m,pinterest,c5")
    ap.add_argument("--old-users", type=int, default=20000)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    cutoffs = [1, 5, 10]
    report = {"card": card(), "cutoffs": cutoffs, "shapes": {}}
    print(report["card"], flush=True)
    for name in args.shapes.split(","):
        n_users, n_items, density = SHAPES[name]
        train, test, neg = loo_data(n_users, n_items, density, seed=1)
        ev = EvaluatorNegativeItemSample(test, neg, cutoff_list=cutoffs, verbose=False)
        # the first users only, for the old path (and the new one on the same users, to compare the results)
        n_old = min(args.old_users, n_users)
        test_sub = sps.csr_matrix(test[:n_old])
        test_sub.resize((n_users, n_items))
        ev_new_sub = EvaluatorNegativeItemSample(test_sub, neg, cutoff_list=cutoffs, verbose=False)
        ev_old_sub = OldPathEvaluator(test_sub, neg, cutoff_list=cutoffs, verbose=False)
        block = min([1000, int(4 * 1e9 * 8 / 64 / n_items), len(ev.users_to_evaluate)])
        shape = {"n_users": n_users, "n_items": n_items, "train_nnz": int(train.nnz),
                 "candidates": int(ev._cand_ptr[-1]), "block_size": block, "old_users": len(ev_old_sub.users_to_evaluate), "models": {}}
        for label, rec in models(name, train, seed=2):
            ev.evaluateRecommender(rec)  # warm-up: device copies, caches, module loads
            ev_old_sub.evaluateRecommender(rec)
            r = {"new_users_per_s": [], "old_users_per_s": [], "max_rel_diff_old_new": [], "score_kernel_s": [], "score_block_gather_s": []}
            for _ in range(args.rounds):
                t, _ = wall(lambda: ev.evaluateRecommender(rec))
                r["new_users_per_s"].append(len(ev.users_to_evaluate) / t)
                t, res_old = wall(lambda: ev_old_sub.evaluateRecommender(rec))
                r["old_users_per_s"].append(len(ev_old_sub.users_to_evaluate) / t)
                res_new, _ = ev_new_sub.evaluateRecommender(rec)
                r["max_rel_diff_old_new"].append(max_rel_diff(res_new, res_old[0]))
                r["score_kernel_s"].append(scoring_time(ev, rec, block, by_block=False))
                r["score_block_gather_s"].append(scoring_time(ev, rec, block, by_block=True))
            shape["models"][label] = r
            print(name, label, json.dumps(r), flush=True)
            del rec
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
