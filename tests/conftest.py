import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a)")


@pytest.fixture(scope="session", autouse=True)
def _built():
    """Builds libqwgpu.so / the oracle if the artefacts are missing (they are git-ignored)."""
    import __graft_entry__ as g
    if not (os.path.exists(os.path.join(ROOT, "quickwit_b200", "libqwgpu.so"))
            and os.path.exists(os.path.join(ROOT, "oracle", "libqworacle.so"))):
        g.build()
    yield


@pytest.fixture(scope="session")
def gpu_ctx():
    from quickwit_b200.service import SearcherContext
    ctx = SearcherContext(0)
    yield ctx
    ctx.close()
