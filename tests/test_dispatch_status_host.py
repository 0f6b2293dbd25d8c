"""The status each stateless dispatch entry point returns for a faulty argument, without a GPU.

Every case here is refused before the library makes any CUDA call, so the fake device addresses below are never
touched and no kernel is launched (checked through ovrfsr_kernel_launches).  A zero constant block or NISConfig makes
EASU, the fused kernel and both NIS passes refuse the scale (OVRFSR_ERR_UNSUPPORTED) before they reach the device;
cases that would reach a launch are not run.  The table pins both the statuses and the order of the checks: which
fault wins when an argument has two."""
import ctypes as C

import pytest

from openvr_fsr_b200 import _lib as L

SRC, DST = 0x7f0000000000, 0x7f0000100000
W, H = 64, 32
BPP = {L.FORMAT_RGBA16F: 8, L.FORMAT_RGBA32F: 16, L.FORMAT_RGB32F: 12}


def _img(fmt=L.FORMAT_RGBA8, addr=SRC, w=W, h=H, pitch=None, samples=1):
    bpp = BPP.get(fmt & L.FORMAT_LAYOUT_MASK, 4)
    return L.Image(addr, w, h, w * bpp * samples if pitch is None else pitch, fmt, 1, 0, samples)


def _dst(fmt=L.FORMAT_RGBA8, addr=DST, **kw):
    return _img(fmt, addr=addr, **kw)


# each fault: the source, the destination, whether the constants / NISConfig pointer is null, and the pass flags
FAULTS = {
    "none": dict(),
    "src_missing": dict(src=None),
    "src_data_null": dict(src=_img(addr=0)),
    "dst_missing": dict(dst=None),
    "dst_data_null": dict(dst=_dst(addr=0)),
    "consts_null": dict(null=True),
    "src_zero_width": dict(src=_img(w=0)),
    "dst_zero_height": dict(dst=_dst(h=0)),
    "src_unknown_format": dict(src=_img(9)),
    "dst_unknown_format": dict(dst=_dst(9)),
    "dst_srgb_tag": dict(dst=_dst(L.FORMAT_RGBA8 | L.FORMAT_SRGB_BIT)),
    "src_rgb32f": dict(src=_img(L.FORMAT_RGB32F)),
    "dst_rgb32f": dict(dst=_dst(L.FORMAT_RGB32F)),
    "dst_bgra8": dict(dst=_dst(L.FORMAT_BGRA8)),
    "dst_bgrx8": dict(dst=_dst(L.FORMAT_BGRX8)),
    "src_msaa": dict(src=_img(samples=4)),
    "src_msaa_pitch_short": dict(src=_img(samples=4, pitch=W * 4)),
    "dst_msaa": dict(dst=_dst(samples=2)),
    "src_pitch_short": dict(src=_img(pitch=W * 4 - 4)),
    "src_pitch_not_texel": dict(src=_img(L.FORMAT_RGBA16F, pitch=W * 8 + 4)),
    "src_base_misaligned": dict(src=_img(addr=SRC + 2)),
    "dst_pitch_short": dict(dst=_dst(pitch=W * 4 - 4)),
    "dst_pitch_not_texel": dict(dst=_dst(L.FORMAT_RGBA32F, pitch=W * 16 + 8)),
    "dst_base_misaligned": dict(dst=_dst(L.FORMAT_RGBA16F, addr=DST + 4)),
    "ten_bit_src_eight_bit_dst": dict(src=_img(L.FORMAT_RGB10A2)),
    "eight_bit_src_ten_bit_dst": dict(dst=_dst(L.FORMAT_RGB10A2)),
    "ten_bit_src_float_dst": dict(src=_img(L.FORMAT_RGB10A2), dst=_dst(L.FORMAT_RGBA16F)),
    "pass_flags_unknown": dict(src=_img(L.FORMAT_RGBA16F), flags=4),
    "pass_flags_unorm_src": dict(flags=L.PASS_SRTM_IN),
    "pass_flags_float_src": dict(src=_img(L.FORMAT_RGBA32F), flags=L.PASS_SRTM_IN | L.PASS_SRTM_OUT),
    "size_mismatch": dict(dst=_dst(w=W + 1)),
    "size_smaller": dict(dst=_dst(w=W - 1)),
    "src_array": dict(src=_img(L.FORMAT_RGBA8 | L.FORMAT_ARRAY_BIT)),
    "dst_array": dict(dst=_dst(L.FORMAT_RGBA8 | L.FORMAT_ARRAY_BIT)),
    # two faults: the one checked first wins
    "consts_null_and_src_rgb32f": dict(src=_img(L.FORMAT_RGB32F), null=True),
    "src_array_and_consts_null": dict(src=_img(L.FORMAT_RGBA8 | L.FORMAT_ARRAY_BIT), null=True),
    "src_array_and_src_rgb32f": dict(src=_img(L.FORMAT_RGB32F | L.FORMAT_ARRAY_BIT)),
    "src_rgb32f_and_dst_bgra8": dict(src=_img(L.FORMAT_RGB32F), dst=_dst(L.FORMAT_BGRA8)),
    "src_rgb32f_and_pitch_short": dict(src=_img(L.FORMAT_RGB32F, pitch=W * 4)),
    "dst_bgra8_and_pitch_short": dict(dst=_dst(L.FORMAT_BGRA8, pitch=W * 4 - 4)),
    "dst_msaa_pitch_short": dict(dst=_dst(samples=2, pitch=W * 4)),
    "pass_flags_unknown_and_dst_bgra8": dict(src=_img(L.FORMAT_RGBA16F), dst=_dst(L.FORMAT_BGRA8), flags=4),
    "pass_flags_unorm_src_and_size_mismatch": dict(dst=_dst(w=W + 1), flags=L.PASS_SRTM_OUT),
}


def _u32(n, null):
    return None if null else (C.c_uint32 * n)()


def _cfg(null):
    return None if null else C.create_string_buffer(256)


def _ref(img):
    return None if img is None else C.byref(img)


# the ten entry points: (call, takes pass flags); CAS runs its sharpen-only variant
ENTRIES = {
    "easu": (lambda s, d, n, f, m: L.lib().ovrfsr_dispatch_fsr_easu(s, d, _u32(24, n), m, None), False),
    "easu_ex": (lambda s, d, n, f, m: L.lib().ovrfsr_dispatch_fsr_easu_ex(s, d, _u32(24, n), m, f, None), True),
    "rcas": (lambda s, d, n, f, m: L.lib().ovrfsr_dispatch_fsr_rcas(s, d, _u32(12, n), m, None), False),
    "rcas_ex": (lambda s, d, n, f, m: L.lib().ovrfsr_dispatch_fsr_rcas_ex(s, d, _u32(12, n), m, f, None), True),
    "fused": (lambda s, d, n, f, m: L.lib().ovrfsr_dispatch_fsr_fused(s, d, _u32(24, n), _u32(12, False), m, None), False),
    "cas": (lambda s, d, n, f, m: L.lib().ovrfsr_dispatch_cas(s, d, _u32(8, n), 1, m, None), False),
    "nis_scaler": (lambda s, d, n, f, m: L.lib().ovrfsr_dispatch_nis_scaler(s, d, _cfg(n), m, None), False),
    "nis_scaler_ex": (lambda s, d, n, f, m: L.lib().ovrfsr_dispatch_nis_scaler_ex(s, d, _cfg(n), m, f, None), True),
    "nis_sharpen": (lambda s, d, n, f, m: L.lib().ovrfsr_dispatch_nis_sharpen(s, d, _cfg(n), m, None), False),
    "nis_sharpen_ex": (lambda s, d, n, f, m: L.lib().ovrfsr_dispatch_nis_sharpen_ex(s, d, _cfg(n), m, f, None), True),
}


# One column per entry of ENTRIES, in order (easu, easu_ex, rcas, rcas_ex, fused, cas, nis_scaler, nis_scaler_ex,
# nis_sharpen, nis_sharpen_ex): I = OVRFSR_ERR_INVALID, U = OVRFSR_ERR_UNSUPPORTED, - = not run (the case reaches a
# kernel launch, passes pass flags to an entry without them, or has an array image that only fused and CAS refuse
# without asking the runtime about it).  Recorded from the library before the FSR and NIS dispatches shared their
# checks; the same in both math modes.
EXPECTED = {
    "none":                                   "UU--U-UUUU",
    "src_missing":                            "IIIIIIIIII",
    "src_data_null":                          "IIIIIIIIII",
    "dst_missing":                            "IIIIIIIIII",
    "dst_data_null":                          "IIIIIIIIII",
    "consts_null":                            "IIIIIIIIII",
    "src_zero_width":                         "IIIIIIIIII",
    "dst_zero_height":                        "IIIIIIIIII",
    "src_unknown_format":                     "UUUUUUUUUU",
    "dst_unknown_format":                     "UUUUUUUUUU",
    "dst_srgb_tag":                           "UUUUUUUUUU",
    "src_rgb32f":                             "UUUUUUUUUU",
    "dst_rgb32f":                             "UUUUUUUUUU",
    "dst_bgra8":                              "UUUUUUUUUU",
    "dst_bgrx8":                              "UUUUUUUUUU",
    "src_msaa":                               "UUUUUUUUUU",
    "src_msaa_pitch_short":                   "IIIIIIUUUU",
    "dst_msaa":                               "UUUUUUUUUU",
    "src_pitch_short":                        "IIIIIIIIII",
    "src_pitch_not_texel":                    "IIIIIIIIII",
    "src_base_misaligned":                    "IIIIIIIIII",
    "dst_pitch_short":                        "IIIIIIIIII",
    "dst_pitch_not_texel":                    "IIIIIIIIII",
    "dst_base_misaligned":                    "IIIIIIIIII",
    "ten_bit_src_eight_bit_dst":              "UUUUUUUUUU",
    "eight_bit_src_ten_bit_dst":              "UUUUUUUUUU",
    "ten_bit_src_float_dst":                  "UU--U-UUUU",
    "pass_flags_unknown":                     "-I-I---I-I",
    "pass_flags_unorm_src":                   "-U-U---U-U",
    "pass_flags_float_src":                   "-U-----U-U",
    "size_mismatch":                          "UUIIUUUUII",
    "size_smaller":                           "UUIIUUUUII",
    "src_array":                              "----UU----",
    "dst_array":                              "----UU----",
    "consts_null_and_src_rgb32f":             "IIIIIIIIII",
    "src_array_and_consts_null":              "----II----",
    "src_array_and_src_rgb32f":               "----UU----",
    "src_rgb32f_and_dst_bgra8":               "UUUUUUUUUU",
    "src_rgb32f_and_pitch_short":             "IIIIIIUUUU",
    "dst_bgra8_and_pitch_short":              "IIIIIIUUUU",
    "dst_msaa_pitch_short":                   "IIIIIIUUUU",
    "pass_flags_unknown_and_dst_bgra8":       "-U-U---U-U",
    "pass_flags_unorm_src_and_size_mismatch": "-U-U---U-U",
}
CODES = {L.OK: "O", L.ERR_INVALID: "I", L.ERR_UNSUPPORTED: "U", L.ERR_CUDA: "C"}


def status(entry, fault, mode):
    """the letter of the status `entry` returns for `fault` (CODES), or '-' where the entry takes no pass flags"""
    call, takes_flags = ENTRIES[entry]
    f = FAULTS[fault]
    flags = f.get("flags", 0)
    if flags and not takes_flags:
        return "-"
    rc = call(_ref(f.get("src", _img())), _ref(f.get("dst", _dst())), f.get("null", False), flags, mode)
    return CODES.get(rc, str(rc))


def test_table_covers_every_fault_and_entry():
    assert set(EXPECTED) == set(FAULTS)
    assert all(len(row) == len(ENTRIES) for row in EXPECTED.values())


@pytest.mark.parametrize("mode", [L.MATH_STRICT, L.MATH_FAST], ids=["strict", "fast"])
@pytest.mark.parametrize("fault", list(FAULTS))
def test_dispatch_status(built_lib, fault, mode):
    before = L.lib().ovrfsr_kernel_launches()
    got = "".join("-" if want == "-" else status(entry, fault, mode) for entry, want in zip(ENTRIES, EXPECTED[fault]))
    assert got == EXPECTED[fault], dict(zip(ENTRIES, got))
    assert L.lib().ovrfsr_kernel_launches() == before
