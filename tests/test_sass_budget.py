"""Static instruction budget of the two strict kernels of the bench.py headline (tools/sass_per_pixel.py, cuobjdump, no
GPU needed).  The bounds sit a few percent above the counts of the current build, so a change that brings back the
dropped operations fails here by name:
  * EASU filter loop: 459 per pixel (474 while the feature blend started from `0 +`, the tap offset 0 was `0 - ppy`
    and the store address was formed from (x, y) for every pixel);
  * RCAS decode: 23.6 per pixel (27.7 while the paired tile still decoded alpha);
  * RCAS filter and stores: 144.2 per pixel (158.4 with the factors of 4 in the limiter and the `a == 0` selects in the
    reciprocals; those selects were the kernel's FSETPs)."""
import importlib.util
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]


@pytest.fixture(scope="module")
def counts(built_lib):
    import shutil
    if not (shutil.which("cuobjdump") or Path("/usr/local/cuda/bin/cuobjdump").exists()):
        pytest.skip("cuobjdump not installed")
    spec = importlib.util.spec_from_file_location("sass_per_pixel", ROOT / "tools" / "sass_per_pixel.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.per_pixel(built_lib)


def test_strict_easu_filter_loop_budget(counts):
    assert counts["easu_filter"]["per_px"] <= 459 * 1.02


def test_strict_rcas_decode_budget(counts):
    assert counts["rcas_decode"]["per_px"] <= 23.6 * 1.03


def test_strict_rcas_filter_budget(counts):
    assert counts["rcas_rest"]["per_px"] <= 144.2 * 1.03
    assert counts["rcas_total_static"]["mix"]["FSETP"] <= 2
