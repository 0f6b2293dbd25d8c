"""The kernel ledger of the built library (cuobjdump -elf + cu++filt, no GPU): the shipped __global__ functions are
exactly the instantiations the launch switches of csrc/kernels.inc produce, family by family.  A new template axis,
format or kernel changes this set, and this test then fails until tests/kernel_ledger.py (and with it the variant
matrix, tests/test_gpu_variant_matrix.py) learns it."""
import pytest

from tests import kernel_ledger as kl


@pytest.fixture(scope="module")
def shipped(built_lib):
    try:
        return kl.ledger(built_lib)
    except FileNotFoundError as e:
        pytest.skip(f"{e} not installed")


def test_both_demangler_spellings_give_one_key():
    cufilt = "void ovrfsr::strict_math::easu_kernel<(int)4, (int)2, (int)72, (bool)0, (bool)1, (bool)1>" \
             "(ovrfsr::strict_math::EasuArgs, CUtensorMap_st, ovrfsr::strict_math::ArrayIO)"
    cxa = "void ovrfsr::strict_math::easu_kernel<4, 2, 72, false, true, true>" \
          "(ovrfsr::strict_math::EasuArgs, CUtensorMap_st, ovrfsr::strict_math::ArrayIO)"
    assert kl.normalise(cufilt) == kl.normalise(cxa) == ("strict", "easu_kernel", (4, 2, 72, 0, 1, 1))
    assert kl.normalise("void ovrfsr::fast_math::rcas_rcp_selftest_kernel(unsigned int*)") == ("fast", "rcas_rcp_selftest_kernel", ())
    assert kl.normalise("(anonymous namespace)::repitch_rows_kernel(unsigned char*, unsigned long, const unsigned char*, "
                        "unsigned long, unsigned int, unsigned int)") == ("", "repitch_rows_kernel", ())
    assert kl.normalise("void at::native::elementwise_kernel<128, 2>(int, at::native::Fn)") is None
    with pytest.raises(ValueError):  # a template axis the ledger does not know
        kl.normalise("void ovrfsr::fast_math::nis_sharpen_kernel<(int)0, (int)0, (bool)0, (bool)1>(ovrfsr::fast_math::NisArgs)")


def test_expected_keys_match_the_closed_forms():
    assert kl.family_counts(kl.expected_keys()) == kl.FAMILY_COUNTS
    assert sum(kl.FAMILY_COUNTS.values()) == 677


def test_shipped_kernels_are_the_expected_instantiations(shipped):
    got, want = set(shipped), kl.expected_keys()
    assert not got - want, "shipped but not in the ledger's matrix:\n" + "\n".join(kl.describe(k) for k in sorted(got - want))
    assert not want - got, "in the ledger's matrix but not shipped:\n" + "\n".join(kl.describe(k) for k in sorted(want - got))
    assert kl.family_counts(got) == kl.FAMILY_COUNTS


def test_resolve_ships_no_two_sample_vector_variant_for_4_byte_formats(shipped):
    resolve = sorted(args for (_, k, args) in shipped if k == "resolve_msaa_kernel")
    assert len(resolve) == 14
    assert (kl.RGBA8, 2) not in resolve and (kl.RGB10A2, 2) not in resolve
    assert (kl.RGBA16F, 2) in resolve and (kl.RGBA32F, 2) in resolve
