"""scikit-learn's NMF run the way MatrixFactorization/NMFRecommender.py:33-60 runs it (TEST INFRASTRUCTURE; the product never
imports this module).  The reference passes alpha=0.0, which scikit-learn >= 1.2 no longer accepts; its default alpha_W = 0
is the same model, so the call below leaves it out.  The installed scikit-learn is the specification (DESIGN.md §7)."""
import warnings

import numpy as np
import scipy.sparse as sps

SOLVERS = {"multiplicative_update": "mu", "coordinate_descent": "cd"}


def nmf_reference(URM, num_factors=100, l1_ratio=0.5, solver="multiplicative_update", init_type="random", beta_loss="frobenius",
                  random_seed=None, dtype=np.float32):
    """(USER_factors [n_users, f], ITEM_factors [n_items, f], n_iter of fit, n_iter of transform) of NMFRecommender.fit on
    URM cast to `dtype`.  The transform count comes from the same _fit_transform(X, H=components_, update_H=False) call
    that NMF.transform makes."""
    from sklearn.decomposition import NMF
    from sklearn.exceptions import ConvergenceWarning
    X = sps.csr_matrix(URM, dtype=dtype)
    model = NMF(n_components=num_factors, init=init_type, l1_ratio=l1_ratio, solver=SOLVERS[solver], beta_loss=beta_loss,
                random_state=random_seed)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        model.fit(X)
        W, _, n_iter_transform = model._fit_transform(X, H=model.components_, update_H=False)
    return W, model.components_.T.copy(), int(model.n_iter_), int(n_iter_transform)


def solve_from(URM, W, H, solver, beta_loss, max_iter, tol, update_h):
    """One sklearn solve in float64 from the given W [n_users, f] and H [f, n_items] (copied): _fit_multiplicative_update or
    _fit_coordinate_descent with no regularisation.  Returns (W, H, n_iter)."""
    from sklearn.decomposition._nmf import _fit_coordinate_descent, _fit_multiplicative_update
    X = sps.csr_matrix(URM, dtype=np.float64)
    W = np.array(W, dtype=np.float64, order="C")
    H = np.array(H, dtype=np.float64, order="C")
    if SOLVERS.get(solver, solver) == "cd":
        return _fit_coordinate_descent(X, W, H, tol=tol, max_iter=max_iter, update_H=update_h)
    return _fit_multiplicative_update(X, W, H, beta_loss=beta_loss, max_iter=max_iter, tol=tol, update_H=update_h)
