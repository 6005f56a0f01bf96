import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def _ensure_native_library():
    """The built .so normally travels with the tree; if a checkout arrives without it and nvcc is on
    the box, build it once (test infrastructure only -- the product itself never builds or falls back)."""
    lib = ROOT / "pixelsplat_b200" / "_C" / "libpixelsplat_b200.so"
    if not lib.exists():
        import shutil
        import subprocess
        if shutil.which("nvcc") or Path("/usr/local/cuda/bin/nvcc").exists():
            subprocess.run(["make", "-C", str(ROOT / "pixelsplat_b200" / "csrc"), "-j8", "-s"], check=False)


_ensure_native_library()


@pytest.fixture(scope="session", autouse=True)
def _build_oracle():
    from oracle import raster_oracle
    raster_oracle.build()
