import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

os.environ.setdefault("B200DP_OFFLINE", "1")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")
    config.addinivalue_line("markers", "multigpu: needs >= 2 CUDA devices")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        ngpu = torch.cuda.device_count() if torch.cuda.is_available() else 0
    except Exception:
        ngpu = 0
    for item in items:
        if "multigpu" in item.keywords and ngpu < 2:
            item.add_marker(pytest.mark.skip(reason="needs >= 2 GPUs"))
        elif "gpu" in item.keywords and ngpu < 1:
            item.add_marker(pytest.mark.skip(reason="needs a GPU"))


@pytest.fixture
def hvd_single():
    """Fresh single-process runtime (no launcher env)."""
    import distributed_torch_horovod_gcp_b200.torch as hvd
    saved = {k: os.environ.pop(k) for k in list(os.environ)
             if k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "LOCAL_WORLD_SIZE") or
             k.startswith("HOROVOD_")}
    hvd.shutdown()
    hvd.init()
    yield hvd
    hvd.shutdown()
    os.environ.update(saved)
