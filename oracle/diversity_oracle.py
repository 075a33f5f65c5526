"""CPU restatement of DIVERSITY_SIMILARITY (Base/Evaluation/metrics.py:719-775, Diversity_similarity) as the reference's
evaluators compute it.  TEST INFRASTRUCTURE ONLY.

`evaluate_scores_with_diversity` is oracle/evaluator_oracle.py's `evaluate_scores` plus the metric: the same users, the same
ranking of a dense score matrix (Base/BaseRecommender.py:164-207) and, per user and cutoff, a literal float64 transcription
of `Diversity_similarity.add_recommendations` on `recommended_items[0:cutoff]` (Evaluator.py)."""
import numpy as np
import scipy.sparse as sps

from oracle.evaluator_oracle import evaluate_scores


def diversity_similarity(D, recommended_items_ids):
    """One user's term of Diversity_similarity.add_recommendations (metrics.py:733-741), transcribed literally on a float64
    D: the row loop stops at L - 2, and a list of L <= 1 items divides the Python float 0.0 by 0 (ZeroDivisionError)."""
    current_recommended_items_diversity = 0.0
    for item_index in range(len(recommended_items_ids) - 1):
        item_id = recommended_items_ids[item_index]
        item_other_diversity = D[item_id, recommended_items_ids]
        item_other_diversity[item_index] = 0.0
        current_recommended_items_diversity += np.sum(item_other_diversity)
    return current_recommended_items_diversity / (len(recommended_items_ids) * (len(recommended_items_ids) - 1))


def recommendation_lists(URM_train, URM_test, S, cutoff_list, min_ratings_per_user=1, exclude_seen=True, ignore_items=None,
                         ignore_users=None, URM_test_negative=None):
    """(evaluated users, their recommendation lists of up to max(cutoff_list) items), chosen and ranked exactly as
    evaluator_oracle.evaluate_scores does."""
    URM_train = sps.csr_matrix(URM_train)
    T = sps.csr_matrix(URM_test, dtype=np.float64).copy()
    T.eliminate_zeros()
    T.sort_indices()
    n_users, n_items = T.shape
    ignore_items = np.array([] if ignore_items is None else ignore_items, dtype=np.int64)
    ignore_users_arr = np.array([] if ignore_users is None else ignore_users, dtype=np.int64)
    pruned = sps.csc_matrix(T.copy())  # Evaluator.py:137-152, :199
    for i in ignore_items:
        pruned.data[pruned.indptr[i]:pruned.indptr[i + 1]] = 0
    pruned.eliminate_zeros()
    users = np.flatnonzero(np.ediff1d(sps.csr_matrix(pruned).indptr) >= min_ratings_per_user)  # :204-214
    users = np.array(sorted(set(users.tolist()) - set(ignore_users_arr.tolist())), dtype=np.int64)  # :216-222
    rank_items = None
    if URM_test_negative is not None:  # Evaluator.py:497-499
        rank_items = sps.csr_matrix(T.astype(bool)) + sps.csr_matrix(sps.csr_matrix(URM_test_negative).astype(bool))
        rank_items.eliminate_zeros()
    max_cutoff = max(cutoff_list)
    lists = []
    for u in users:
        s = np.array(S[u], dtype=np.float64)
        if exclude_seen:
            s[URM_train.indices[URM_train.indptr[u]:URM_train.indptr[u + 1]]] = -np.inf  # BaseRecommender.py:166-169
        s[ignore_items] = -np.inf  # :192-193
        if rank_items is not None:  # the non-candidates score -inf (BaseSimilarityMatrixRecommender.py:84-90)
            keep = np.zeros(n_items, bool)
            keep[rank_items.indices[rank_items.indptr[u]:rank_items.indptr[u + 1]]] = True
            s[~keep] = -np.inf
        order = np.lexsort((np.arange(n_items), -s))[:max_cutoff]
        lists.append(order[np.isfinite(s[order])])  # :203-207
    return users, lists


def evaluate_scores_with_diversity(URM_train, URM_test, S, cutoff_list, item_diversity_matrix, **kw):
    """evaluate_scores(...) with DIVERSITY_SIMILARITY added for every cutoff: the mean over the evaluated users of
    diversity_similarity(D, list[0:cutoff]), D = item_diversity_matrix in float64 (a short list raises, as in the
    reference).  Each cutoff value counts once, like the per-cutoff metric objects of the reference."""
    D = np.asarray(item_diversity_matrix, dtype=np.float64)
    users, lists = recommendation_lists(URM_train, URM_test, S, cutoff_list, **kw)
    div = {}
    for c in cutoff_list:
        total = 0.0
        for r in lists:
            total += diversity_similarity(D, r[:c])
        div[c] = total / len(users) if len(users) else 0.0
    out = evaluate_scores(URM_train, URM_test, S, cutoff_list, **kw)
    for c in out:
        out[c]["DIVERSITY_SIMILARITY"] = float(div[c])
    return out
