"""The reference's run_example_usage.py (run_example_usage.py:1-83) on this package: same flow -- build a split, create
the evaluators, fit a few recommenders with fit(**hyperparameters), evaluate, save and reload a model -- with the hot
loops on the GPU and a synthetic data set instead of the Movielens1M reader (no network here).

    python examples/usage_example.py
"""
import os
import sys

import numpy as np
import scipy.sparse as sps

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from recsys2019_deeplearning_evaluation_b200.evaluation import EvaluatorHoldout  # noqa: E402
from recsys2019_deeplearning_evaluation_b200.knn import ItemKNNCBFRecommender, ItemKNN_CFCBF_Hybrid_Recommender  # noqa: E402
from recsys2019_deeplearning_evaluation_b200.nonpersonalized import TopPop  # noqa: E402
from recsys2019_deeplearning_evaluation_b200.recommenders import (EASE_R_Recommender, IALSRecommender, ItemKNNCFRecommender,  # noqa: E402
                                                                  MatrixFactorization_BPR_Cython, P3alphaRecommender,
                                                                  RP3betaRecommender, SLIM_BPR_Cython)
from recsys2019_deeplearning_evaluation_b200.synth import synth_urm  # noqa: E402


def leave_k_out(URM_all, k, rng):
    """Per user, k random interactions go to the held-out matrix (what DataSplitter_leave_k_out does for k_out_value=k)."""
    URM_all = sps.csr_matrix(URM_all)
    hold = np.zeros(URM_all.nnz, bool)
    for u in range(URM_all.shape[0]):
        s, e = URM_all.indptr[u], URM_all.indptr[u + 1]
        if e - s > k + 1:
            hold[rng.choice(np.arange(s, e), size=k, replace=False)] = True
    coo = URM_all.tocoo()
    mk = lambda m: sps.csr_matrix((coo.data[m], (coo.row[m], coo.col[m])), shape=URM_all.shape, dtype=np.float32)  # noqa: E731
    return mk(~hold), mk(hold)


def main():
    rng = np.random.default_rng(0)
    URM_all = synth_urm(6040, 3706, 0.0447, seed=42, values="ratings", popularity=0.8)   # Movielens1M shape
    ICM_genres = synth_urm(3706, 18, 0.09, seed=7, values="binary")
    URM_train_all, URM_test = leave_k_out(URM_all, 1, rng)
    URM_train, URM_validation = leave_k_out(URM_train_all, 1, rng)
    evaluator_validation = EvaluatorHoldout(URM_validation, cutoff_list=[5], exclude_seen=False)
    evaluator_test = EvaluatorHoldout(URM_test, cutoff_list=[5, 10, 20], exclude_seen=False)

    recommender = TopPop(URM_train)
    recommender.fit()
    print("Result of TopPop is:\n" + evaluator_validation.evaluateRecommender(recommender)[1])

    for cls, fit_kw in ((P3alphaRecommender, dict(topK=100, alpha=0.5)), (RP3betaRecommender, dict(topK=100, alpha=0.5, beta=0.3)),
                        (ItemKNNCFRecommender, dict(topK=100, shrink=50, similarity="cosine", feature_weighting="TF-IDF")),
                        (EASE_R_Recommender, dict(l2_norm=2000.0)),
                        (IALSRecommender, dict(epochs=10, num_factors=64, alpha=5.0, reg=1e-2)),
                        (SLIM_BPR_Cython, dict(epochs=20, topK=100, sgd_mode="adagrad", learning_rate=1e-3, random_seed=42)),
                        (MatrixFactorization_BPR_Cython, dict(epochs=50, num_factors=64, batch_size=1000, learning_rate=5e-3,
                                                              sgd_mode="adagrad", random_seed=42,
                                                              evaluator_object=evaluator_validation, validation_every_n=10,
                                                              validation_metric="MAP", stop_on_validation=True,
                                                              lower_validations_allowed=2))):
        recommender = cls(URM_train)
        recommender.fit(**fit_kw)
        print("Result of {} is:\n".format(recommender.RECOMMENDER_NAME) + evaluator_validation.evaluateRecommender(recommender)[1])

    recommender = ItemKNNCBFRecommender(URM_train, ICM_genres)
    recommender.fit(topK=100, similarity="cosine")
    print("Result of ItemKNNCBF is:\n" + evaluator_validation.evaluateRecommender(recommender)[1])
    recommender = ItemKNN_CFCBF_Hybrid_Recommender(URM_train, ICM_genres)
    recommender.fit(topK=100, similarity="cosine")
    print("Result of ItemKNN_CFCBF_Hybrid is:\n" + evaluator_validation.evaluateRecommender(recommender)[1])

    # save, reload into a fresh object, evaluate on the test split (run_example_usage.py:70-83)
    folder = "result_experiments/usage_example/"
    recommender.save_model(folder, file_name="hybrid_model")
    reloaded = ItemKNN_CFCBF_Hybrid_Recommender(URM_train, ICM_genres)
    reloaded.load_model(folder, file_name="hybrid_model")
    print("Test result of the reloaded hybrid is:\n" + evaluator_test.evaluateRecommender(reloaded)[1])


if __name__ == "__main__":
    main()
