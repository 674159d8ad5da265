"""pytest wiring: `-m "not gpu"` runs on the CPU-only build container, `-m gpu` on an H100."""
import os
import sys

import pytest

REPO = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
PKG = os.path.join(REPO, "second.pytorch_b200")
for p in (REPO, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def oracle():
    """the CPU oracle `spconv` package (test infrastructure), loaded under an alias."""
    from b2second import loader
    return loader.oracle_spconv()


@pytest.fixture(scope="session")
def product():
    """the CUDA `spconv` drop-in; loading fails loudly if libb2second.so is missing."""
    from b2second import loader
    mod = loader.product_spconv()
    mod._lib.load()
    return mod


@pytest.fixture(scope="session")
def out_dir():
    d = os.path.join(REPO, "gpurun_out")
    os.makedirs(d, exist_ok=True)
    return d


@pytest.fixture(scope="module")
def ref_env():
    # the reference imports its plugin by the name `spconv`: make that name the CPU oracle for this module's
    # tests (other test modules in the same process use the CUDA drop-in under that name), then restore
    saved = {k: v for k, v in sys.modules.items() if k == "spconv" or k.startswith("spconv.")}
    for k in saved:
        del sys.modules[k]
    saved_path = list(sys.path)
    from b2second import loader as _loader
    sys.path[:] = [p for p in sys.path if os.path.abspath(p) != os.path.abspath(_loader.PRODUCT_DIR)] + \
        [_loader.PRODUCT_DIR]
    from b2second import loader, refcompat
    refcompat.install(loader.ORACLE_DIR)
    import spconv
    assert getattr(spconv, "__oracle__", False)
    yield spconv
    for k in [k for k in sys.modules if k == "spconv" or k.startswith("spconv.")]:
        del sys.modules[k]
    sys.modules.update(saved)
    sys.path[:] = saved_path


