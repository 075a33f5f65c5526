import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (select with -m gpu)")


# Under `pytest tests -x -q -m gpu` a failure hides everything collected after it.  The headline path goes
# first (similarity kernel and its reference goldens, then the SGD trainers), the remaining files keep their
# alphabetical order behind them.
_ORDER = ["test_similarity_gpu", "test_golden_gpu", "test_scale_parity_gpu", "test_mf_gpu", "test_slim_gpu",
          "test_recommenders_gpu", "test_euclidean_gpu", "test_graph_gpu", "test_ials", "test_ease_gpu"]


_LAST = ["test_next_rows_gpu"]  # the SURVEY.md 8(f).4 trainers: behind everything on the hot path


def _rank(item):
    name = os.path.splitext(os.path.basename(str(item.fspath)))[0]
    if name in _LAST:
        return len(_ORDER) + 1 + _LAST.index(name)
    return _ORDER.index(name) if name in _ORDER else len(_ORDER)


def pytest_collection_modifyitems(config, items):
    items.sort(key=_rank)  # stable: order inside a file and among the unlisted files is unchanged
    # GPU tests are selected with `-m gpu`; without a device they are skipped rather than failed when
    # someone runs the whole suite on a CPU box.
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
