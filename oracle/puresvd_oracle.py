"""scikit-learn's randomized_svd run the way MatrixFactorization/PureSVDRecommender.py:36-55 runs it (TEST INFRASTRUCTURE; the
product never imports this module).  The installed scikit-learn is the specification (DESIGN.md §7)."""
import numpy as np
import scipy.sparse as sps


def puresvd_reference(URM, num_factors=100, random_seed=None, dtype=np.float32):
    """(USER_factors [n_users, k'], ITEM_factors [n_items, k'], s [k']) of PureSVDRecommender.fit on URM cast to `dtype`:
    U, Sigma, VT = randomized_svd(URM, n_components=num_factors, random_state=random_seed), USER_factors = U,
    ITEM_factors = (diag(Sigma) VT)^T."""
    from sklearn.utils.extmath import randomized_svd
    X = sps.csr_matrix(URM, dtype=dtype)
    U, Sigma, VT = randomized_svd(X, n_components=num_factors, random_state=random_seed)
    return U, (sps.diags(Sigma) @ VT).T, Sigma
