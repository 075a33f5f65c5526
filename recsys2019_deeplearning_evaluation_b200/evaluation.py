"""Host-side mirror of the reference's hold-out evaluator, with the per-user metric loop on the device.

`EvaluatorHoldout(URM_test, cutoff_list, min_ratings_per_user=1, exclude_seen=True, ignore_items=None,
ignore_users=None).evaluateRecommender(recommender)` -> `(results_dict, results_run_string)` like
Base/Evaluation/Evaluator.py:152-461: same constructor logic (users with too few test interactions and ignored users
are skipped, :182-225), same block loop (:420-455), same result keys (`EvaluatorMetrics`, :20-45) and result string
(:119-135).  What changes is where the work happens: for every block of users the recommender's masked score block
and its top-`max_cutoff` table stay on the device (recommenders.BaseRecommender._masked_scores_device / _topn_device)
and `b200_eval_accumulate_device` (csrc/eval.cu) reduces all per-user metrics of :336-366 into device accumulators;
the host only combines the final sums and the per-item recommendation counters (O(n_items) once per evaluation).

`EvaluatorNegativeItemSample` (Evaluator.py:466-578) walks the same blocks of users, but scores and ranks only each user's
candidate list (test items + sampled negatives) with the csrc/score.cu candidate kernels before the same accumulate kernel.

With a `diversity_object` (metrics.py:719-775: any object with an `item_diversity_matrix`, such as `Diversity_similarity`
below or the reference's own class) both evaluators add DIVERSITY_SIMILARITY, the 23rd metric: the top-left
n_items x n_items block of the matrix is uploaded once per evaluator and device, and `b200_eval_diversity_device` reduces
each block's lists next to the accumulate kernel.

Any other recommender object -- the reference's own `BaseRecommender` subclasses, such as the neural wrappers or
`GlobalEffects` -- is a *foreign* recommender.  It needs only the reference methods the reference evaluator calls:
`_compute_item_score(user_id_array, items_to_compute=None)`, `get_URM_train()`, `set_items_to_ignore` and
`reset_items_to_ignore`.  Its host score blocks are uploaded and ranked on the device (fp32 blocks on the fp32 top-N keys,
fp64 blocks on 96-bit fp64 keys, csrc/score.cu) and go to the same accumulate kernel (see
`EvaluatorHoldout.evaluateRecommender`).
"""
import ctypes

import numpy as np
import scipy.sparse as sps

from . import _lib
from .recommenders import BaseRecommender

# order of Base/Evaluation/Evaluator.py:20-45
METRIC_NAMES = ["PRECISION", "PRECISION_RECALL_MIN_DEN", "RECALL", "MAP", "MAP_MIN_DEN", "MRR", "NDCG", "F1", "HIT_RATE",
                "ARHR_ALL_HITS", "NOVELTY", "AVERAGE_POPULARITY", "DIVERSITY_MEAN_INTER_LIST", "DIVERSITY_HERFINDAHL",
                "COVERAGE_ITEM", "COVERAGE_ITEM_HIT", "ITEMS_IN_GT", "COVERAGE_USER", "COVERAGE_USER_HIT", "USERS_IN_GT",
                "DIVERSITY_GINI", "SHANNON_ENTROPY"]
_SLOT = dict(PRECISION=0, PRECISION_RECALL_MIN_DEN=1, RECALL=2, MAP=3, MAP_MIN_DEN=4, MRR=5, NDCG=6, HIT_RATE=7, ARHR_ALL_HITS=8,
             NOVELTY=9, AVERAGE_POPULARITY=10, USERS_WITH_RECS=11, N_USERS=12, DIVERSITY_SIMILARITY=13, SHORT_LISTS=14)
_NACC = 16
# with a diversity object, the reference's EvaluatorMetrics order puts DIVERSITY_SIMILARITY after AVERAGE_POPULARITY
_METRIC_NAMES_DIVERSITY = METRIC_NAMES[:METRIC_NAMES.index("AVERAGE_POPULARITY") + 1] + ["DIVERSITY_SIMILARITY"] + \
    METRIC_NAMES[METRIC_NAMES.index("AVERAGE_POPULARITY") + 1:]


class Diversity_similarity(object):
    """metrics.py:719-731: holds the dense item-item diversity matrix D for the evaluators' `diversity_object` argument.
    For a recommendation list r of length L >= 2 a user's value is
    sum_{a <= L-2} sum_{b <= L-1, b != a} D[r_a, r_b] / (L (L - 1)) (the last row is skipped, its column is not); the
    metric is the mean over the evaluated users.  A list shorter than 2 items makes the evaluation raise
    ZeroDivisionError, as the reference's 0.0 / 0 does."""

    def __init__(self, item_diversity_matrix):
        assert np.all(item_diversity_matrix >= 0.0) and np.all(item_diversity_matrix <= 1.0), \
            "item_diversity_matrix contains value greated than 1.0 or lower than 0.0"
        self.item_diversity_matrix = item_diversity_matrix


def get_result_string(results_run, n_decimals=7):
    """Evaluator.py:119-135."""
    output_str = ""
    for cutoff in results_run.keys():
        output_str += "CUTOFF: {} - ".format(cutoff)
        for metric in results_run[cutoff].keys():
            output_str += "{}: {:.{n_decimals}f}, ".format(metric, results_run[cutoff][metric], n_decimals=n_decimals)
        output_str += "\n"
    return output_str


def _remove_item_interactions(URM, item_list):
    """Evaluator.py:137-152."""
    URM = sps.csc_matrix(URM.copy())
    for item_index in item_list:
        URM.data[URM.indptr[int(item_index)]:URM.indptr[int(item_index) + 1]] = 0
    URM.eliminate_zeros()
    return sps.csr_matrix(URM)


def _ideal_dcg(URM_test, cutoffs):
    """[n_users, n_cutoffs] float64: dcg of each user's test ratings sorted descending, cut at every cutoff
    (metrics.py:268, :277-279).  One-off preprocessing of the test set, vectorised."""
    n_users = URM_test.shape[0]
    lens = np.diff(URM_test.indptr)
    rows = np.repeat(np.arange(n_users), lens)
    order = np.lexsort((-URM_test.data.astype(np.float64), rows))
    rel = URM_test.data.astype(np.float64)[order]
    pos = np.arange(len(rel)) - np.repeat(URM_test.indptr[:-1], lens)
    terms = (np.power(2.0, rel) - 1.0) / np.log2(pos + 2.0)
    out = np.zeros((n_users, len(cutoffs)))
    for k, c in enumerate(cutoffs):
        out[:, k] = np.bincount(rows, weights=np.where(pos < c, terms, 0.0), minlength=n_users)
    return out


def _foreign_scores(recommender_object, user_id_array, n_items, items_to_compute=None):
    """One `_compute_item_score` call of a foreign recommender, as the reference's `recommend` makes it: the block as a
    C-contiguous float32 or float64 array of shape (len(user_id_array), n_items).  Other real dtypes become float64."""
    block = np.asarray(recommender_object._compute_item_score(user_id_array, items_to_compute=items_to_compute))
    want = (len(user_id_array), n_items)
    if block.shape != want:
        raise ValueError("{}._compute_item_score returned a score block of shape {}, expected {} (users, n_items)".format(
            type(recommender_object).__name__, block.shape, want))
    if block.dtype.kind not in "biuf":
        raise ValueError("{}._compute_item_score returned scores of dtype {}, expected real numbers".format(
            type(recommender_object).__name__, block.dtype))
    if block.dtype != np.float32 and block.dtype != np.float64:
        block = np.asarray(block, np.float64)
    return np.ascontiguousarray(block)


class EvaluatorHoldout(object):
    EVALUATOR_NAME = "EvaluatorHoldout"

    def __init__(self, URM_test_list, cutoff_list, min_ratings_per_user=1, exclude_seen=True, diversity_object=None,
                 ignore_items=None, ignore_users=None, verbose=True):
        self.verbose = verbose
        if ignore_items is None:  # Evaluator.py:168-174
            self.ignore_items_flag = False
            self.ignore_items_ID = np.array([], dtype=np.int64)
        else:
            self._print("Ignoring {} Items".format(len(ignore_items)))
            self.ignore_items_flag = True
            self.ignore_items_ID = np.array(ignore_items, dtype=np.int64)
        self.cutoff_list = list(cutoff_list)
        self.max_cutoff = max(self.cutoff_list)
        if self.max_cutoff > 1024:
            raise ValueError("EvaluatorHoldout: cutoffs above 1024 are not supported on the CUDA path")
        self.min_ratings_per_user = min_ratings_per_user
        self.exclude_seen = exclude_seen
        if isinstance(URM_test_list, list):
            raise ValueError("List of URM_test not supported")  # :187
        # :184 keeps the test matrix as passed (ignored items stay relevant); Items_In_GT.__init__ (metrics.py:375) drops
        # its explicit zeros in place before the first user is scored
        self.URM_test = sps.csr_matrix(URM_test_list.copy(), dtype=np.float32)
        self.URM_test.eliminate_zeros()
        self.URM_test.sort_indices()
        self.n_users, self.n_items = self.URM_test.shape
        self._div = None  # the diversity matrix D on the host, then (_div_device) on the device
        if diversity_object is not None:
            D = np.asarray(diversity_object.item_diversity_matrix)
            if D.ndim != 2 or D.shape[0] < self.n_items or D.shape[1] < self.n_items:
                raise ValueError("{}: diversity_object.item_diversity_matrix must be a dense 2-D array of at least {} x {} "
                                 "(n_items), got shape {}".format(self.EVALUATOR_NAME, self.n_items, self.n_items, D.shape))
            # item ids index D, so only its top-left n_items x n_items block is read; float32 stays float32, any other
            # dtype is read as float64
            self._div = np.ascontiguousarray(D[:self.n_items, :self.n_items],
                                             np.float32 if D.dtype == np.float32 else np.float64)
        pruned = _remove_item_interactions(URM_test_list, self.ignore_items_ID)  # :199
        mask = np.ediff1d(pruned.indptr) >= min_ratings_per_user  # :204-208
        if not np.all(mask):
            self._print("Ignoring {} ({:4.1f}%) Users that have less than {} test interactions".format(
                np.sum(mask), 100 * np.sum(np.logical_not(mask)) / len(mask), min_ratings_per_user))
        users = np.arange(self.n_users)[mask]
        if ignore_users is not None:  # :216-222
            self._print("Ignoring {} Users".format(len(ignore_users)))
            self.ignore_users_ID = np.array(ignore_users, dtype=np.int64)
            users = np.array(sorted(set(users.tolist()) - set(int(u) for u in ignore_users)), dtype=np.int64)
        else:
            self.ignore_users_ID = np.array([], dtype=np.int64)
        self.users_to_evaluate = list(users)
        self._lib = _lib.load()
        self._dev = None
        self._d_div = None

    def _print(self, string):
        if self.verbose:
            print("{}: {}".format(self.EVALUATOR_NAME, string))

    def _div_device(self, dev):
        """The diversity matrix on the device, uploaded once per evaluator and device (early stopping evaluates often)."""
        import torch
        if self._d_div is None or self._d_div.device != dev:
            self._d_div = None  # free the copy on the old device before the new one is made
            self._d_div = torch.from_numpy(self._div).to(dev)
        return self._d_div

    # ------------------------------------------------------------------------------------------------------------
    def _device_state(self, URM_train):
        import torch
        dev = torch.device("cuda", torch.cuda.current_device())
        T = self.URM_test
        pop = np.ediff1d(sps.csc_matrix(URM_train).indptr).astype(np.float64)  # metrics.py:629-632 (train zeros eliminated upstream)
        n_inter = pop.sum()
        with np.errstate(divide="ignore", invalid="ignore"):
            nov = np.where(pop > 0, -np.log2(pop / n_inter) / len(pop), 0.0)  # :648-651
        pop_norm = pop / pop.max() if pop.max() > 0 else pop  # :686
        st = dict(
            ptr=torch.from_numpy(np.ascontiguousarray(T.indptr, np.int32)).to(dev),
            idx=torch.from_numpy(np.ascontiguousarray(T.indices, np.int32)).to(dev),
            val=torch.from_numpy(np.ascontiguousarray(T.data, np.float32)).to(dev),
            cut=torch.from_numpy(np.asarray(self.cutoff_list, np.int32)).to(dev),
            idcg=torch.from_numpy(_ideal_dcg(T, self.cutoff_list)).to(dev),
            nov=torch.from_numpy(nov).to(dev), pop=torch.from_numpy(np.ascontiguousarray(pop_norm, np.float64)).to(dev),
            acc=torch.zeros((len(self.cutoff_list), _NACC), dtype=torch.float64, device=dev),
            rec=torch.zeros((len(self.cutoff_list), self.n_items), dtype=torch.int32, device=dev),
            hit=torch.zeros((len(self.cutoff_list), self.n_items), dtype=torch.int32, device=dev))
        if self._div is not None:
            st["div"] = self._div_device(dev)
        return st

    def _accumulate(self, st, d_users, items, vals, cutoff):
        """Adds one block's [B, cutoff] top-N table to the device accumulators (csrc/eval.cu)."""
        import torch
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        _lib.check(self._lib.b200_eval_accumulate_device(
            d_users.data_ptr(), d_users.shape[0], items.data_ptr(), vals.data_ptr(), cutoff, st["ptr"].data_ptr(),
            st["idx"].data_ptr(), st["val"].data_ptr(), st["cut"].data_ptr(), len(self.cutoff_list), st["idcg"].data_ptr(),
            st["nov"].data_ptr(), st["pop"].data_ptr(), self.n_items, st["acc"].data_ptr(), st["rec"].data_ptr(),
            st["hit"].data_ptr(), stream))
        if "div" in st:
            _lib.check(self._lib.b200_eval_diversity_device(
                items.data_ptr(), vals.data_ptr(), d_users.shape[0], cutoff, st["cut"].data_ptr(), len(self.cutoff_list),
                st["div"].data_ptr(), int(st["div"].dtype == torch.float64), self.n_items, st["acc"].data_ptr(), stream))

    def _evaluate_blocks(self, recommender_object, users, block_size, st):
        """Hold-out evaluation scores whole blocks of users (:426-455)."""
        cutoff = int(min(self.max_cutoff, self.n_items))
        for b0 in range(0, len(users), block_size):
            d_users = recommender_object._users_tensor(users[b0:b0 + block_size])
            scores = recommender_object._masked_scores_device(d_users, remove_seen_flag=self.exclude_seen, items_to_compute=None,
                                                              remove_custom_items_flag=self.ignore_items_flag)
            items, vals = recommender_object._topn_device(scores, cutoff)
            self._accumulate(st, d_users, items, vals, cutoff)

    def _foreign_blocks(self, recommender_object, users, block_size):
        """(users, host score block) of a foreign recommender: one call per block of users, items_to_compute=None (:426-437)."""
        for b0 in range(0, len(users), block_size):
            b_users = users[b0:b0 + block_size]
            yield b_users, _foreign_scores(recommender_object, b_users, self.n_items)

    def _evaluate_foreign(self, recommender_object, users, block_size, st, URM_train):
        """Ranks every host score block of a foreign recommender on the device: upload, seen (the structure of its
        URM_train) and ignored items to -inf, [B, max_cutoff] top-N table, accumulate.  Nothing here waits for the device,
        so the GPU ranks block b while the model scores block b + 1 on the host."""
        import torch
        URM_train = sps.csr_matrix(URM_train)
        if URM_train.shape[0] < self.n_users or URM_train.shape[1] != self.n_items:
            raise ValueError("{}: get_URM_train() has shape {}, the test matrix {}".format(
                self.EVALUATOR_NAME, URM_train.shape, self.URM_test.shape))
        dev = st["ptr"].device
        seen_ptr = seen_idx = keep = None
        if self.exclude_seen:
            seen_ptr, seen_idx = (torch.from_numpy(np.ascontiguousarray(a, np.int32)).to(dev)
                                  for a in (URM_train.indptr, URM_train.indices))
        if self.ignore_items_flag and len(self.ignore_items_ID):
            k = np.ones(self.n_items, np.uint8)
            k[self.ignore_items_ID] = 0
            keep = torch.from_numpy(k).to(dev)
        cutoff = int(min(self.max_cutoff, self.n_items))
        rows = min(block_size, max(len(users), 1))
        items = torch.empty((rows, cutoff), dtype=torch.int32, device=dev)
        vals = torch.empty((rows, cutoff), dtype=torch.float32, device=dev)
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        for b_users, block in self._foreign_blocks(recommender_object, users, block_size):
            nb = len(b_users)
            # non_blocking: torch's blocking host-to-device copy synchronises the stream after the copy; a copy from pageable
            # memory has still consumed the host array when the call returns
            d_users = torch.from_numpy(np.ascontiguousarray(b_users, np.int32)).to(dev, non_blocking=True)
            d_scores = torch.from_numpy(block).to(dev, non_blocking=True)
            f64 = block.dtype == np.float64
            if seen_ptr is not None or keep is not None:
                mask = self._lib.b200_score_mask_f64_device if f64 else self._lib.b200_score_mask_device
                _lib.check(mask(d_users.data_ptr() if seen_ptr is not None else None, nb,
                                seen_ptr.data_ptr() if seen_ptr is not None else None,
                                seen_idx.data_ptr() if seen_idx is not None else None,
                                keep.data_ptr() if keep is not None else None, self.n_items, d_scores.data_ptr(), stream))
            topn = self._lib.b200_score_topn_f64_device if f64 else self._lib.b200_score_topn_device
            _lib.check(topn(d_scores.data_ptr(), nb, self.n_items, cutoff, items.data_ptr(), vals.data_ptr(), stream))
            self._accumulate(st, d_users, items[:nb], vals[:nb], cutoff)

    def evaluateRecommender(self, recommender_object, block_size=None):
        """Evaluator.py:240-288 + :413-461.

        `recommender_object` is one of this package's `BaseRecommender` mirrors, whose score blocks never leave the
        device, or any foreign object with the reference's `_compute_item_score(user_id_array, items_to_compute=None)`,
        `get_URM_train()`, `set_items_to_ignore` and `reset_items_to_ignore`.  A foreign object is called as the reference
        evaluator calls it: `_compute_item_score` once per block of users here (consecutive int64 slices of
        `users_to_evaluate`, items_to_compute=None), once per user in EvaluatorNegativeItemSample; `get_URM_train()` once.
        Its block must be `np.asarray`-able to shape (len(user_id_array), n_items), else ValueError.  float32 blocks are
        ranked in fp32 and float64 blocks in fp64; any other real dtype (ints, bool, float16) is converted with
        `np.asarray(block, np.float64)`, which is exact except for int64 magnitudes above 2^53.  The seen items (the
        structure of `sps.csr_matrix(get_URM_train())`, with exclude_seen) and the ignored items score -inf, and the
        ranking is the package's own: np.lexsort((arange, -s)), ties to the ascending item, +inf first and NaN last, and
        only the finite entries of the first max_cutoff positions are recommendations (DESIGN.md §6c).  The object's own
        `recommend()` is not called (the reference's argpartition leaves its tie order unspecified)."""
        if self.ignore_items_flag:
            recommender_object.set_items_to_ignore(self.ignore_items_ID)
        users = np.asarray(self.users_to_evaluate, dtype=np.int64)
        if block_size is None:  # :422
            block_size = min([1000, int(4 * 1e9 * 8 / 64 / self.n_items), max(len(users), 1)])
        URM_train = recommender_object.get_URM_train()
        st = self._device_state(URM_train)
        if isinstance(recommender_object, BaseRecommender):
            self._evaluate_blocks(recommender_object, users, block_size, st)
        else:
            self._evaluate_foreign(recommender_object, users, block_size, st, URM_train)
        acc, rec, hit = st["acc"].cpu().numpy(), st["rec"].cpu().numpy().astype(np.float64), st["hit"].cpu().numpy().astype(np.float64)
        n_eval = len(users)
        results_dict = {}
        keep = np.ones(self.n_items, dtype=bool)
        keep[self.ignore_items_ID] = False
        gt_items = np.ediff1d(sps.csc_matrix(self.URM_test).indptr) > 0
        gt_items[self.ignore_items_ID] = False
        gt_users = np.ediff1d(self.URM_test.indptr) > 0
        gt_users[self.ignore_users_ID] = False
        names = METRIC_NAMES if self._div is None else _METRIC_NAMES_DIVERSITY
        for k, c in enumerate(self.cutoff_list):
            r = {}
            if n_eval > 0:
                a = acc[k]
                if self._div is not None:
                    if a[_SLOT["SHORT_LISTS"]] > 0:  # metrics.py:741, 0.0 / (L * (L - 1)) for a list of L <= 1 items
                        raise ZeroDivisionError("float division by zero")
                    r["DIVERSITY_SIMILARITY"] = float(a[_SLOT["DIVERSITY_SIMILARITY"]] / n_eval)
                for name in ("PRECISION", "PRECISION_RECALL_MIN_DEN", "RECALL", "MAP", "MAP_MIN_DEN", "MRR", "NDCG", "HIT_RATE",
                             "ARHR_ALL_HITS", "NOVELTY", "AVERAGE_POPULARITY"):
                    r[name] = float(a[_SLOT[name]] / n_eval)
                p_, r_ = r["PRECISION"], r["RECALL"]
                r["F1"] = 2 * (p_ * r_) / (p_ + r_) if p_ + r_ != 0 else 0.0  # Evaluator.py:270-276
                cnt = rec[k][keep]  # metrics.py:305-314
                tot = cnt.sum()
                r["COVERAGE_ITEM"] = float((cnt > 0).sum() / len(cnt))  # :338-342
                r["COVERAGE_ITEM_HIT"] = float((hit[k][keep] > 0).sum() / len(cnt))  # :357-361
                r["ITEMS_IN_GT"] = float(gt_items.sum() / (len(gt_items) - len(self.ignore_items_ID)))  # :383-388
                r["COVERAGE_USER"] = float(a[_SLOT["USERS_WITH_RECS"]] / (self.n_users - len(self.ignore_users_ID)))  # :438-439
                r["COVERAGE_USER_HIT"] = float(a[_SLOT["HIT_RATE"]] / (self.n_users - len(self.ignore_users_ID)))  # :466-467
                r["USERS_IN_GT"] = float(gt_users.sum() / (len(gt_users) - len(self.ignore_users_ID)))  # :408-413
                n = len(cnt)
                srt = np.sort(cnt)
                r["DIVERSITY_GINI"] = float(2 * np.sum((n + 1 - np.arange(1, n + 1)) / (n + 1) * srt / tot)) if tot > 0 else float("nan")  # :503-520
                r["DIVERSITY_HERFINDAHL"] = float(1 - np.sum((cnt / tot) ** 2)) if tot != 0 else float("nan")  # :549-556
                pr = cnt[cnt > 0] / tot if tot > 0 else np.zeros(0)
                r["SHANNON_ENTROPY"] = float(-np.sum(pr * np.log2(pr)))  # :592-608
                couples = n_eval ** 2 - n_eval  # :860-873 (its counter is NOT filtered by ignore_items)
                co = np.sum(rec[k] ** 2) - n_eval * c
                r["DIVERSITY_MEAN_INTER_LIST"] = float((couples - co / c) / couples) if couples > 0 else float("nan")
                results_dict[c] = {name: r[name] for name in names}
            else:
                results_dict[c] = {name: 0.0 for name in names}
        if n_eval == 0:
            self._print("WARNING: No users had a sufficient number of relevant items")
        if self.ignore_items_flag:
            recommender_object.reset_items_to_ignore()
        return results_dict, get_result_string(results_dict)


class EvaluatorNegativeItemSample(EvaluatorHoldout):
    """Base/Evaluation/Evaluator.py:466-578: every user is ranked over HER test items plus her sampled negative items only
    (the protocol of the NeuMF-style experiments).  The reference scores one user at a time (:553-571) over the whole
    catalogue with the other items masked; here blocks of users score and rank their candidates only, on the device:
    `rec._candidate_scores_device` (a ragged array aligned with the candidate CSR) -> `b200_cand_topn_device` (seen and
    ignored candidates -> -inf, the [B, max_cutoff] table of the hold-out path) -> the same accumulate kernel.  Every
    non-candidate scores -inf in the reference's ranking, so its finite prefix -- the recommendation list -- is the same."""
    EVALUATOR_NAME = "EvaluatorNegativeItemSample"

    def __init__(self, URM_test_list, URM_test_negative, cutoff_list, min_ratings_per_user=1, exclude_seen=True,
                 diversity_object=None, ignore_items=None, ignore_users=None, verbose=True):
        super(EvaluatorNegativeItemSample, self).__init__(URM_test_list, cutoff_list, min_ratings_per_user=min_ratings_per_user,
                                                          exclude_seen=exclude_seen, diversity_object=diversity_object,
                                                          ignore_items=ignore_items, ignore_users=ignore_users, verbose=verbose)
        rank = sps.csr_matrix(self.URM_test.astype(bool)) + sps.csr_matrix(sps.csr_matrix(URM_test_negative).astype(bool))  # :497
        rank.eliminate_zeros()
        rank.sort_indices()
        self.URM_items_to_rank = rank
        # the candidate lists in users_to_evaluate order, so that a block of users is a contiguous slice
        cand = rank[np.asarray(self.users_to_evaluate, dtype=np.int64)]
        if cand.nnz >= 2 ** 31:
            raise ValueError("EvaluatorNegativeItemSample: more than 2^31 - 1 candidate items in total")
        self._cand_ptr = np.ascontiguousarray(cand.indptr, np.int32)
        self._cand_idx = np.ascontiguousarray(cand.indices, np.int32)
        self._d_cand = None

    def _get_user_specific_items_to_compute(self, user_id):
        r = self.URM_items_to_rank
        return r.indices[r.indptr[user_id]:r.indptr[user_id + 1]]

    def _foreign_blocks(self, recommender_object, users, block_size):
        """A foreign recommender is called once per user with the user's sorted candidate row as items_to_compute (:553-571);
        the rows are stacked into blocks of block_size users and each full row is ranked, so a non-candidate counts as
        whatever score the model gave it, as in the reference's `recommend`."""
        for b0 in range(0, len(users), block_size):
            b_users = users[b0:b0 + block_size]
            rows = [_foreign_scores(recommender_object, np.atleast_1d(u), self.n_items, self._get_user_specific_items_to_compute(u))
                    for u in b_users]
            yield b_users, rows[0] if len(rows) == 1 else np.concatenate(rows)

    def _cand_device(self, dev):
        """(users, candidate pointer, candidate items) on the device, uploaded once per evaluator."""
        import torch
        if self._d_cand is None or self._d_cand[0].device != dev:
            users = np.asarray(self.users_to_evaluate, dtype=np.int32)
            self._d_cand = tuple(torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (users, self._cand_ptr, self._cand_idx))
        return self._d_cand

    def _evaluate_blocks(self, recommender_object, users, block_size, st):
        import torch
        n = len(users)
        if n == 0:
            return
        dev = st["ptr"].device
        d_users, d_ptr, d_idx = self._cand_device(dev)
        cutoff = int(min(self.max_cutoff, self.n_items))
        starts = np.arange(0, n, block_size)
        longest = int(np.max(self._cand_ptr[np.minimum(starts + block_size, n)] - self._cand_ptr[starts]))
        scores = torch.empty(max(longest, 1), dtype=torch.float32, device=dev)
        items = torch.empty((min(block_size, n), cutoff), dtype=torch.int32, device=dev)
        vals = torch.empty((min(block_size, n), cutoff), dtype=torch.float32, device=dev)
        seen_ptr = seen_idx = ignore = None
        if self.exclude_seen:
            seen_ptr, seen_idx, _ = (t.data_ptr() for t in recommender_object._urm_device())
        if self.ignore_items_flag and len(recommender_object.items_to_ignore_ID):  # BaseRecommender.py:192-193
            mask = np.zeros(self.n_items, np.uint8)
            mask[recommender_object.items_to_ignore_ID] = 1
            ignore = torch.from_numpy(mask).to(dev)
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        for b0 in starts.tolist():
            nb = min(block_size, n - b0)
            b_users, b_ptr = d_users[b0:b0 + nb], d_ptr[b0:b0 + nb + 1]
            recommender_object._candidate_scores_device(b_users, b_ptr, d_idx, scores)
            _lib.check(self._lib.b200_cand_topn_device(
                b_users.data_ptr(), nb, b_ptr.data_ptr(), d_idx.data_ptr(), scores.data_ptr(), seen_ptr, seen_idx,
                ignore.data_ptr() if ignore is not None else None, cutoff, items.data_ptr(), vals.data_ptr(), stream))
            self._accumulate(st, b_users, items[:nb], vals[:nb], cutoff)

