"""Strict RCAS on a UNORM8 source evaluates the limiter with its factors of 4 taken out (fsr_kernels.cuh rcas_filter):
1/mx and 1/(mn-1) instead of 1/(4mx) and 1/(4mn-4), the clamp at -3/4 instead of -3/16, then x0.25 before x sharp.
The lobe depends on the decoded (mn, mx) of each channel only, so every code pair with mn <= mx (32,896 of them) is
checked here in float32, one IEEE rounding per device operation, against the reference's operation order
(ffx_fsr1.h:748-760)."""
import numpy as np

f32 = np.float32


def _channel_lobes():
    v = np.arange(256, dtype=f32) / f32(255.0)  # the exact UNORM8 decode (tests/test_host_logic.py)
    mn, mx = np.meshgrid(v, v, indexing="ij")
    reachable = mn <= mx  # mn and mx are the min and the max of the same four texels
    mn, mx = mn[reachable], mx[reachable]
    assert mn.size == 256 * 257 // 2
    with np.errstate(divide="ignore", invalid="ignore"):
        # reference: rcp.rn of 4mx and 4mn-4 (1/+0 = +inf, and 0 * inf = NaN)
        ref = np.fmax(-(mn * (f32(1) / (f32(4) * mx))), (f32(1) - mx) * (f32(1) / (f32(4) * mn + f32(-4))))
        # device sequence: MUFU.RCP + one Newton step, which gives NaN for +0 (equal to rcp.rn elsewhere, checked on the
        # device by ovrfsr_selftest_rcp)
        def rcp(x):
            return np.where(x == 0, f32(np.nan), f32(1) / x).astype(f32)
        new = np.fmax(-(mn * rcp(mx)), (f32(1) - mx) * rcp(mn + f32(-1)))
    return ref, new


def test_limiter_without_factors_of_four_is_exact_for_every_unorm8_code_pair():
    ref, new = _channel_lobes()
    assert ref.dtype == new.dtype == f32
    assert np.array_equal(np.isnan(ref), np.isnan(new))
    ok = ~np.isnan(ref)
    assert np.array_equal((new[ok] * f32(0.25)).view(np.uint32), ref[ok].view(np.uint32))
    # the clamped lobe before and after x sharp, for sharp values from the API's range and far outside it
    # (x0.25 is applied before x sharp, so a sharp that makes the product subnormal keeps the reference's rounding)
    ref_c = np.fmax(f32(-(0.25 - 1.0 / 16.0)), np.fmin(ref, f32(0)))
    new_c = np.fmax(f32(-4.0 * (0.25 - 1.0 / 16.0)), np.fmin(new, f32(0))) * f32(0.25)
    assert np.array_equal(new_c.view(np.uint32), ref_c.view(np.uint32))
    for sharp in (f32(1.0), f32(0.5358867), f32(0.25), f32(2.0 ** -120), f32(2.0 ** -140), f32(0.0)):
        ref_l, new_l = ref_c * sharp, new_c * sharp
        assert np.array_equal(new_l.view(np.uint32), ref_l.view(np.uint32)), sharp
        assert np.array_equal((f32(4) * new_l + f32(1)).view(np.uint32), (f32(4) * ref_l + f32(1)).view(np.uint32))


def test_every_lobe_operand_is_a_normal_float_or_zero():
    """The identities x4 / x0.25 hold because nothing on the UNORM8 domain is subnormal."""
    ref, new = _channel_lobes()
    for a in (ref, new):
        a = np.abs(a[~np.isnan(a)])
        assert (a[a != 0] >= np.finfo(f32).tiny).all()
