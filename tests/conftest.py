import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# BB_PKG_ROOT points the suite at another build of the package (sanitizer builds: build/asan/out, see build.py)
PKG_ROOT = os.path.abspath(os.environ.get("BB_PKG_ROOT", ROOT))
for p in (ROOT, PKG_ROOT):
    if p in sys.path:
        sys.path.remove(p)
sys.path.insert(0, ROOT)
if PKG_ROOT != ROOT:
    sys.path.insert(0, PKG_ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA GPU (run with -m gpu on an H100 box)")


def _have_module():
    try:
        from blackbird_b200 import _bb  # noqa: F401
        return True
    except Exception:
        return False


if not _have_module():
    # build the native module on demand (seconds when up to date)
    import build as _build

    _build.build()


@pytest.fixture
def bb():
    from blackbird_b200 import _bb

    return _bb
