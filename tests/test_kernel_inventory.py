"""CPU: the tensor-core kernel instantiations compiled into the library are exactly wgmma_variants.ALL_VARIANTS, and each
of them is the expected kernel of at least one GPU test case -- a new instantiation without a test fails here."""
import re
import shutil
import subprocess

import pytest

from tests import test_conv_tcgen05_gpu, test_dcn_gpu, test_gemm_tcgen05_gpu, test_lstm_step_gpu
from tests import wgmma_variants as wv


@pytest.fixture(scope="module")
def so_path():
    from megreader_b200 import build
    return build.build()


def compiled_variants(so_path):
    dump = subprocess.run([shutil.which("cuobjdump"), "-symbols", so_path], check=True, capture_output=True,
                          text=True).stdout
    mangled = sorted(set(re.findall(r"\b_Z\w+", dump)))
    names = subprocess.run([shutil.which("cu++filt")], input="\n".join(mangled), check=True, capture_output=True,
                           text=True).stdout.splitlines()
    return {n for n in map(wv.normalise, names) if re.fullmatch(r"\w+_tcgen05_kernel<[\d,]+>", n)}


@pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None,
                    reason="needs cuobjdump and cu++filt from the CUDA toolkit")
def test_compiled_instantiations_are_the_known_variants(so_path):
    found = compiled_variants(so_path)
    assert len(wv.ALL_VARIANTS) == 20
    assert found == wv.ALL_VARIANTS, ("not in ALL_VARIANTS: %s; not compiled: %s"
                                      % (sorted(found - wv.ALL_VARIANTS), sorted(wv.ALL_VARIANTS - found)))


def test_every_variant_has_a_gpu_case():
    covered = (test_gemm_tcgen05_gpu.VARIANTS | test_conv_tcgen05_gpu.VARIANTS | test_lstm_step_gpu.VARIANTS
               | test_dcn_gpu.VARIANTS)
    assert covered <= wv.ALL_VARIANTS, sorted(covered - wv.ALL_VARIANTS)
    assert covered == wv.ALL_VARIANTS, "no GPU case expects %s" % sorted(wv.ALL_VARIANTS - covered)


def test_dispatch_restatement():
    """spot checks of expected_variant against the host dispatch rules it restates"""
    assert wv.expected_variant("gemm", N=64, transA=0, transB=0) == "gemm_tcgen05_kernel<64,8,0,1>"
    assert wv.expected_variant("gemm", N=65, transA=1, transB=0) == "gemm_tcgen05_kernel<128,6,1,1>"
    assert wv.tma_a_segments(5, 15) == [8, 4, 2, 1]
    assert wv.tma_a_segments(5, 31) is None                      # five segments
    assert wv.tma_a_segments(1, 256) == [128, 128]
    assert wv.tma_a_segments(1, 130, sw=3) is None              # 128 * 3 columns > 256
    fp = dict(H=16, W=128, Cout=64, kh=3, kw=3, ph=1, pw=1)
    assert wv.expected_variant("conv_fprop", env={}, **fp) == "conv_fprop_tcgen05_kernel<64,3,1>"
    assert wv.expected_variant("conv_fprop", env={"MR_CONV_SHALLOW": "0"}, **fp) == "conv_fprop_tcgen05_kernel<64,8,1>"
    assert wv.expected_variant("conv_fprop", env={"MR_CONV_NO_TMA_A": "1"}, **fp) == "conv_fprop_tcgen05_kernel<64,8,0>"
    assert wv.expected_variant("conv_wgrad", H=4, W=72, C=64, kh=1, kw=1) == "conv_wgrad_tcgen05_kernel<64,80,6>"
    assert wv.normalise("void (anonymous namespace)::gemm_tcgen05_kernel<128, 6, 0, 1>(CUtensorMap_st, CUtensorMap_st, "
                        "(anonymous namespace)::GemmArgs)") == "gemm_tcgen05_kernel<128,6,0,1>"
    assert wv.normalise("void <unnamed>::conv_wgrad_tcgen05_kernel<(int)64, (int)80, (int)6>(CUtensorMap_st)") \
        == "conv_wgrad_tcgen05_kernel<64,80,6>"
