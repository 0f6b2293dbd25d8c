"""The numpy restatement of FsrEasuF in tests/easu_direction.py against the oracle, and the threshold content it
measures: bit for bit on every output pixel of every case and of the corner images, and each case's promised number of
pixels whose dir^2 sits within 2 ulps of EASU's direction threshold 2^-15, with both branches taken among them."""
import numpy as np
import pytest

from tests import easu_direction as ed
from tests.cases import corner_images


def _tag(fmt):
    return fmt if fmt in (ed.BGRA8, ed.RGB10A2, ed.BGRX8) else None


def _restated_vs_oracle(src, fmt, iw, ih, scale):
    from oracle import pyoracle as po
    ow, oh = po.output_size(iw, ih, scale)
    uc = po.upscale_constants(0, True, iw, ih, ow, oh, radius=2.0)  # every group inside: the filter everywhere
    pix, dir2, zro = ed.easu(src, fmt, uc.words(), ow, oh)
    want = po.easu(src, ow, oh, uc, out_dtype=np.float32, src_fmt=_tag(fmt))[..., :3]
    bad = np.argwhere(pix.view(np.uint32) != want.view(np.uint32))
    assert len(bad) == 0, f"{len(bad)} channels differ, first at (y, x, ch) = {tuple(bad[0])}: " \
                          f"{pix[tuple(bad[0])]!r} vs {want[tuple(bad[0])]!r}"
    return dir2, zro


@pytest.mark.parametrize("name", sorted(ed.CASES))
def test_restatement_matches_oracle_and_case_sits_on_threshold(name):
    fmt, iw, ih, scale, _, kind, _, min_near = ed.CASES[name]
    dir2, zro = _restated_vs_oracle(ed.case_source(name), fmt, iw, ih, scale)
    near, near_zro, near_dir = ed.near_threshold(dir2, zro)
    print(f"{name}: {near} pixels within 2 ulps of 2^-15 ({near_zro} zro, {near_dir} normalised) of {dir2.size}")
    assert near >= min_near, f"{name}: {near} near-threshold pixels, promised {min_near}"
    if min_near:
        assert near_zro and near_dir, f"{name}: one branch only among the near-threshold pixels"
    if kind == "flat":
        assert zro.all(), f"{name}: luma is flat up to decode rounding, so dir^2 is far below 2^-15 everywhere"
    else:
        assert zro.any() and not zro.all(), f"{name}: the oracle takes one branch everywhere"


@pytest.mark.parametrize("iw,ih,scale", [(33, 47, 0.75), (40, 24, 0.9), (21, 35, 0.59)])
def test_restatement_matches_oracle_on_corner_images(iw, ih, scale):
    for name, img in corner_images(iw, ih).items():
        _restated_vs_oracle(img, ed.RGBA8, iw, ih, scale)


def test_float_ramp_luma_is_exact():
    """the FP32 ramp's construction: luma is c + G to the last bit, so every feature's lE - lA is the chosen step"""
    src = ed.float_ramp(64, 40, ed.RGBA32F, 1)
    luma = src[..., 2] * np.float32(0.5) + (src[..., 0] * np.float32(0.5) + src[..., 1])
    assert np.array_equal(luma, np.float32(ed.CHROMA_C) + src[..., 1])
    i = np.arange(1, 39)
    same_period = (i - 1) // ed.PERIOD == (i + 1) // ed.PERIOD
    d = luma[i + 1, 0] - luma[i - 1, 0]
    assert np.all(d[same_period] == np.float32(ed.K_STEP * ed.Q))
    assert np.ptp(src[..., 0]) > 0.01  # the chroma swings while luma holds
