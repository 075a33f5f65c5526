"""Development timing of both evaluators on foreign recommenders (objects that are not this package's mirrors) on one GPU:
    python tools/dev_foreign_eval_bench.py [--out FILE.json] [--legs holdout,negative] [--rounds R] [--ref-users N]
Shapes: hold-out on the C3 shape (138 000 x 27 000, 0.535 %; each interaction goes to the test set with probability 0.2),
and negative sampling on a Pinterest-like 55 187 x 9 916 shape (one test item and 100 sampled negatives per user).
Models, all scoring on the host with numpy:
  * MF fp32 / MF fp64: U[users] @ V.T with f = 64 seeded random factors (the reference's MF classes hold fp64 factors);
    with items_to_compute, the other items score -inf, as the reference's models do;
  * precomputed: one precomputed fp32 block returned for every call, so the evaluator's own cost is all that is left.
For each (leg, model), `--rounds` times: the total evaluateRecommender time (host clock around the call, which ends in a
device synchronise), the time spent inside _compute_item_score, and the evaluator overhead per user (the difference over
the evaluated users).  For comparison: a numpy restatement of the reference's per-block `recommend` (seen items -> -inf,
argpartition + argsort of the top max_cutoff) plus a per-user metric loop (precision, recall, MAP, nDCG, MRR and hit
rate per cutoff; the reference computes more metrics per user) on the same blocks of the first `--ref-users` users, time
per user with the scoring excluded.  And the host-to-device copy alone of one full block (pageable, as the evaluator makes
it; fp32 and fp64), to see what share of the evaluator's time the upload takes.  The card's name and power limit are
read in the same run."""
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

from recsys2019_deeplearning_evaluation_b200.evaluation import EvaluatorHoldout, EvaluatorNegativeItemSample
from recsys2019_deeplearning_evaluation_b200.synth import CONFIGS, synth_urm

CUTOFFS = [1, 5, 10, 20, 50, 100]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0 or not r.stdout.strip():
        raise RuntimeError("nvidia-smi failed: %s" % r.stdout)
    return r.stdout.strip().splitlines()[0]


class Timed(object):
    """A foreign recommender around a score function; counts the time spent inside _compute_item_score."""

    def __init__(self, URM_train, score_fn):
        self.URM_train = URM_train
        self.score_fn = score_fn
        self.score_s = 0.0

    def get_URM_train(self):
        return self.URM_train.copy()

    def set_items_to_ignore(self, items_to_ignore):
        self.items_to_ignore_ID = np.array(items_to_ignore, dtype=np.int64)

    def reset_items_to_ignore(self):
        self.items_to_ignore_ID = np.array([], dtype=np.int64)

    def _compute_item_score(self, user_id_array, items_to_compute=None):
        t0 = time.perf_counter()
        s = self.score_fn(user_id_array)
        if items_to_compute is not None:
            out = np.full(s.shape, -np.inf, dtype=s.dtype)
            out[:, items_to_compute] = s[:, items_to_compute]
            s = out
        self.score_s += time.perf_counter() - t0
        return s


def mf(n_users, n_items, dtype, seed):
    rng = np.random.default_rng(seed)
    U = (rng.standard_normal((n_users, 64)) * 0.1).astype(dtype)
    V = (rng.standard_normal((n_items, 64)) * 0.1).astype(dtype)
    return lambda users: U[users] @ V.T


def precomputed(n_items, rows, seed):
    block = np.random.default_rng(seed).standard_normal((rows, n_items)).astype(np.float32)
    return lambda users: block[:len(users)]


def holdout_data(seed):
    """C3 (synth.CONFIGS); every interaction goes to the test set with probability 0.2."""
    X = synth_urm(*CONFIGS["C3"], seed=seed, values="ratings")
    rng = np.random.default_rng(seed + 1)
    to_test = rng.random(X.nnz) < 0.2
    coo = X.tocoo()
    def part(m):
        return sps.csr_matrix((coo.data[m], (coo.row[m], coo.col[m])), shape=X.shape)
    return part(~to_test), part(to_test)


def negative_data(seed):
    n_users, n_items = 55187, 9916
    rng = np.random.default_rng(seed)
    train = synth_urm(n_users, n_items, 0.0027, seed=seed, popularity=0.8)
    rows = np.arange(n_users)
    test = sps.csr_matrix((np.ones(n_users, np.float32), (rows, rng.integers(0, n_items, n_users))), shape=(n_users, n_items))
    neg_cols = rng.integers(0, n_items, (n_users, 100)).ravel()
    neg = sps.csr_matrix((np.ones(len(neg_cols), np.float32), (np.repeat(rows, 100), neg_cols)), shape=(n_users, n_items))
    return train, test, neg


def reference_restatement(ev, score_fn, train, n_users_ref, block_size, negative):
    """Host time per user of the reference's ranking (per-block recommend: seen -> -inf, argpartition + argsort) and a
    per-user metric loop, scoring excluded; on the first n_users_ref evaluated users."""
    users = np.asarray(ev.users_to_evaluate[:n_users_ref], dtype=np.int64)
    T = ev.URM_test
    max_cutoff = max(CUTOFFS)
    t_rank = t_metric = 0.0
    for b0 in range(0, len(users), block_size):
        b_users = users[b0:b0 + block_size]
        if negative:  # one call per user, stacked
            R = ev.URM_items_to_rank
            rows = []
            for u in b_users:
                s = score_fn(np.atleast_1d(u))
                keep = np.zeros(s.shape[1], bool)
                keep[R.indices[R.indptr[u]:R.indptr[u + 1]]] = True
                s = np.where(keep, s, -np.inf)
                rows.append(s)
            scores = np.concatenate(rows)
        else:
            scores = score_fn(b_users)
        t0 = time.perf_counter()
        scores = np.array(scores, copy=True)
        for i, u in enumerate(b_users):  # BaseRecommender._remove_seen_on_scores
            scores[i, train.indices[train.indptr[u]:train.indptr[u + 1]]] = -np.inf
        part = np.argpartition(-scores, max_cutoff - 1, axis=1)[:, :max_cutoff]  # BaseRecommender.recommend
        part_scores = scores[np.arange(len(b_users))[:, None], part]
        order = np.argsort(-part_scores, axis=1)
        ranking = part[np.arange(len(b_users))[:, None], order]
        lists = [ranking[i][np.isfinite(scores[i, ranking[i]])] for i in range(len(b_users))]
        t1 = time.perf_counter()
        acc = np.zeros((len(CUTOFFS), 6))
        for i, u in enumerate(b_users):  # Evaluator._compute_metrics_on_recommendation_list
            rel = T.indices[T.indptr[u]:T.indptr[u + 1]]
            is_rel = np.in1d(lists[i], rel, assume_unique=True)
            for k, c in enumerate(CUTOFFS):
                r = is_rel[:c]
                L = max(len(r), 1)
                p_at_k = r * np.cumsum(r, dtype=np.float64) / (1 + np.arange(len(r)))
                dcg = np.sum(r / np.log2(np.arange(len(r)) + 2))
                idcg = np.sum(1 / np.log2(np.arange(min(len(rel), c)) + 2))
                hits = np.flatnonzero(r)
                acc[k] += (r.sum() / L, r.sum() / max(len(rel), 1), p_at_k.sum() / L, dcg / idcg if idcg else 0.0,
                           1.0 / (hits[0] + 1) if len(hits) else 0.0, float(r.any()))
        t_metric += time.perf_counter() - t1
        t_rank += t1 - t0
    return {"users": len(users), "rank_s_per_user": t_rank / len(users), "metric_loop_s_per_user": t_metric / len(users)}


def upload_ms(rows, n_items, dtype, reps=20):
    """Device time of the evaluator's pageable host-to-device copy of one [rows, n_items] block."""
    block = np.random.default_rng(0).standard_normal((rows, n_items)).astype(dtype)
    dev = torch.device("cuda", torch.cuda.current_device())
    torch.from_numpy(block).to(dev, non_blocking=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        torch.from_numpy(block).to(dev, non_blocking=True)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps * 1e3


def run_leg(ev, train, models, rounds, ref_users, negative):
    n_eval = len(ev.users_to_evaluate)
    block = min([1000, int(4 * 1e9 * 8 / 64 / ev.n_items), max(n_eval, 1)])
    out = {"n_users_evaluated": n_eval, "block_size": block, "models": {},
           "upload_ms_per_block": {"fp32": upload_ms(block, ev.n_items, np.float32), "fp64": upload_ms(block, ev.n_items, np.float64)}}
    print("upload", json.dumps(out["upload_ms_per_block"]), flush=True)
    for label, fn in models:
        rec = Timed(train, fn)
        ev.evaluateRecommender(rec)  # warm-up: module loads, device copies
        r = {"total_s": [], "score_s": [], "overhead_us_per_user": []}
        for _ in range(rounds):
            rec.score_s = 0.0
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ev.evaluateRecommender(rec)  # ends in a device-to-host copy of the accumulators
            torch.cuda.synchronize()
            t = time.perf_counter() - t0
            r["total_s"].append(t)
            r["score_s"].append(rec.score_s)
            r["overhead_us_per_user"].append((t - rec.score_s) / n_eval * 1e6)
        r["reference_restatement"] = reference_restatement(ev, fn, train, min(ref_users, n_eval), block, negative)
        out["models"][label] = r
        print(label, json.dumps(r), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--legs", default="holdout,negative")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--ref-users", type=int, default=20000)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this tool measures the GPU path; it needs a CUDA device"
    report = {"card": card(), "cutoffs": CUTOFFS, "legs": {}}
    print(report["card"], flush=True)
    legs = args.legs.split(",")
    if "holdout" in legs:
        train, test = holdout_data(seed=1)
        ev = EvaluatorHoldout(test, CUTOFFS, verbose=False)
        n_users, n_items = train.shape
        models = [("MF fp32", mf(n_users, n_items, np.float32, 2)), ("MF fp64", mf(n_users, n_items, np.float64, 2)),
                  ("precomputed", precomputed(n_items, 1000, 3))]
        report["legs"]["holdout_C3"] = run_leg(ev, train, models, args.rounds, args.ref_users, negative=False)
        del ev, train, test
    if "negative" in legs:
        train, test, neg = negative_data(seed=4)
        ev = EvaluatorNegativeItemSample(test, neg, CUTOFFS, verbose=False)
        n_users, n_items = train.shape
        models = [("MF fp32", mf(n_users, n_items, np.float32, 5)), ("MF fp64", mf(n_users, n_items, np.float64, 5)),
                  ("precomputed", precomputed(n_items, 1, 6))]
        report["legs"]["negative_55K"] = run_leg(ev, train, models, args.rounds, args.ref_users, negative=True)
    txt = json.dumps(report, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(txt)
    print(txt)


if __name__ == "__main__":
    main()
