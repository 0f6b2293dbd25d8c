"""The CHECKER under AddressSanitizer + UndefinedBehaviorSanitizer: every pass of the restated oracle on small ragged
images (1x1 up to 64x24, every format, up- and down-scale factors) must run clean -- an out-of-bounds read in the
oracle would otherwise be able to 'agree' with anything.  The float sources run a second time with about one word in
16 +-inf or a NaN (quiet and signalling, with payloads) into every target format, RCAS also on the source itself (the
encode tests/srtm_oracle.py ends in), with float-cast-overflow among the checks: a texel-derived NaN or infinity that
reached an (int) / (uint8_t) cast without a saturate in front of it would be undefined behaviour, and the checker's
bits would then depend on the compiler.  Skipped where no compiler here ships the sanitizer runtimes.

The numpy restatements (the MSAA resolve, the tone map of tests/srtm_oracle.py) are held to the same on non-finite
input: no NaN or infinity reaches an integer cast (numpy's "invalid value encountered in cast")."""
import warnings
import shutil
import subprocess
from pathlib import Path

import pytest

ORACLE = Path(__file__).resolve().parents[1] / "oracle"


def test_oracle_runs_clean_under_asan_ubsan():
    built = False
    for cc in ("gcc", "/usr/bin/gcc", "cc", "clang"):
        path = shutil.which(cc) or (cc if Path(cc).exists() else None)
        if not path:
            continue
        r = subprocess.run(["make", "-C", str(ORACLE), "-B", "selfcheck", f"SANCC={path}"], capture_output=True, text=True)
        if r.returncode == 0:
            built = True
            break
    if not built:
        pytest.skip("no compiler with the ASan/UBSan runtimes available")
    out = subprocess.run([str(ORACLE / "selfcheck_asan")], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-4000:]
    assert "configurations ok" in out.stdout


def _nonfinite(shape, dtype, seed):
    import numpy as np
    rng = np.random.default_rng(seed)
    a = rng.uniform(-0.5, 7.5, shape).astype(dtype)
    hit = rng.random(shape) < 0.1
    a[hit] = rng.choice(np.array([np.inf, -np.inf, np.nan], dtype=dtype), int(hit.sum()))
    return a


def test_numpy_restatements_cast_no_nonfinite_value():
    import numpy as np
    from oracle import frontend as fe
    from oracle import pyoracle as po
    from tests import srtm_oracle as so
    with warnings.catch_warnings():
        warnings.filterwarnings("ignore", message="invalid value encountered in (add|subtract|multiply|divide)")  # IEEE
        warnings.filterwarnings("error", message="invalid value encountered in cast")
        for dtype, fmt in ((np.float16, po.FMT_RGBA16F), (np.float32, po.FMT_RGBA32F)):
            ms = _nonfinite((9, 4 * 11, 4), dtype, fmt)
            assert np.isnan(fe.resolve_msaa(ms, 4, fmt)).any()
            src = _nonfinite((13, 17, 4), dtype, fmt + 1)
            uc = po.upscale_constants(0, True, 17, 13, 23, 17, radius=0.4)
            sc = po.sharpen_constants(0, True, 17, 13, radius=0.4)
            for out in (np.uint8, np.float16, np.float32):
                so.easu(src, 23, 17, uc, out_dtype=out, srtm_in=True, srtm_out=True)
                so.rcas(src, sc, out_dtype=out, srtm_in=True, srtm_out=True)
        # the resolve's UNORM encodes: NaN stores 0 and +-inf saturates, as the kernels' stores
        f = np.array([[[np.nan, np.inf, -np.inf, 0.5]]], dtype=np.float32)
        assert fe._encode(f, po.FMT_RGBA8).tolist() == [[[0, 255, 0, 128]]]
