"""CPU: how SLIM_BPR_Cython.fit(train_with_sparse_weights=None) picks between the dense and the row-sparse tree mode."""
from recsys2019_deeplearning_evaluation_b200.slim_bpr_epoch import sparse_weights_for_device


def test_none_picks_the_tree_mode_only_when_the_dense_mode_does_not_fit():
    n = 100_000
    need = 8 * n * n  # S plus get_S's buffer, both n x n fp32; a symmetric S is allocated in full too
    for symmetric in (True, False):
        assert sparse_weights_for_device(None, n, need, symmetric) is False
        assert sparse_weights_for_device(None, n, need + 1, symmetric) is False
        assert sparse_weights_for_device(None, n, need - 1, symmetric) is True
        assert sparse_weights_for_device(None, 200_000, 80 * 2 ** 30, symmetric) is True
        assert sparse_weights_for_device(None, 3_706, 80 * 2 ** 30, symmetric) is False


def test_explicit_choices_are_kept():
    for symmetric in (True, False):
        assert sparse_weights_for_device(True, 10, 2 ** 40, symmetric) is True
        assert sparse_weights_for_device(False, 10 ** 6, 0, symmetric) is False
