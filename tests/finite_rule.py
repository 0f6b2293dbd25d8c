"""The host statement of OVRFSR_FLAG_FINITE's two maps (include/ovrfsr.h), for the tests that hold the kernels to it.

finite_in   every channel of a float source texel: NaN -> +0, +-inf -> +-65504, every finite value as it is.
finite_out  every channel of a float image's stored pixel: NaN -> +0, +-inf -> +-(the destination's largest finite
            value).  Applied to a stored FP16 / FP32 word this equals the kernels' clamp-then-round: a value beyond
            the largest finite one rounds to +-inf, and one in (65504, 65520) already rounds to 65504.
Both leave UNORM arrays alone."""
import numpy as np

FP16_MAX = 65504.0


def finite_in(a):
    a = np.asarray(a)
    if a.dtype not in (np.float16, np.float32):
        return a
    out = np.where(np.isnan(a), a.dtype.type(0), a)
    return np.where(np.isinf(out), np.copysign(a.dtype.type(FP16_MAX), out), out).astype(a.dtype)


def finite_out(a):
    a = np.asarray(a)
    if a.dtype not in (np.float16, np.float32):
        return a
    big = np.finfo(a.dtype).max
    out = np.where(np.isnan(a), a.dtype.type(0), a)
    return np.where(np.isinf(out), np.copysign(big, out), out).astype(a.dtype)


def fp16_store(x):
    """the kernels' finite-out before an FP16 store of binary32 values x: clamp to +-65504, then round to nearest"""
    x = np.asarray(x, dtype=np.float32)
    return np.where(np.isnan(x), np.float32(0), np.clip(x, -FP16_MAX, FP16_MAX)).astype(np.float16)
