import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

GOLDEN = ROOT / "tests" / "golden"

# no pretrained checkpoints exist offline: the tests run the real architectures on seeded random weights, which the
# product refuses to do unless asked (weights.resolve_checkpoint)
os.environ.setdefault("FADTK_SYNTHETIC", "1")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a GPU machine)")


def _has_gpu() -> bool:
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture(scope="session")
def engine():
    from fadtk_b200 import _native
    return _native.engine(max_examples=int(os.environ.get("FADTK_MAX_EXAMPLES", "512")))


@pytest.fixture(scope="session")
def vgg_state():
    from fadtk_b200 import weights
    return weights.synthetic_vggish_state(0)


@pytest.fixture(scope="session")
def vgg_engine(engine, vgg_state):
    from fadtk_b200 import weights
    engine.vggish_load(weights.pack_vggish(vgg_state))
    return engine
