"""CPU: the tensor-core kernel instantiations compiled into the library are exactly wgmma_variants.ALL_VARIANTS, and each
of them is the expected kernel of at least one GPU test case -- a new instantiation without a test fails here.  The same
for the CTC kernels (ctc_variants) and the streaming kernels of csrc/nn_kernels.cu (nn_variants)."""
import os
import re
import shutil
import subprocess

import pytest

from tests import ctc_variants as cv
from tests import nn_variants as nv
from tests import test_conv_tcgen05_gpu, test_ctc_variants_gpu, test_dcn_gpu, test_gemm_tcgen05_gpu, test_lstm_step_gpu
from tests import test_decode_gpu, test_nn_kernels_gpu, test_nn_streaming_gpu
from tests import wgmma_variants as wv


@pytest.fixture(scope="module")
def so_path():
    from megreader_b200 import build
    return build.build()


def compiled_kernels(so_path):
    dump = subprocess.run([shutil.which("cuobjdump"), "-symbols", so_path], check=True, capture_output=True,
                          text=True).stdout
    mangled = sorted(set(re.findall(r"\b_Z\w+", dump)))
    return subprocess.run([shutil.which("cu++filt")], input="\n".join(mangled), check=True, capture_output=True,
                          text=True).stdout.splitlines()


def compiled_variants(so_path):
    return {n for n in map(wv.normalise, compiled_kernels(so_path)) if re.fullmatch(r"\w+_tcgen05_kernel<[\d,]+>", n)}


@pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None,
                    reason="needs cuobjdump and cu++filt from the CUDA toolkit")
def test_compiled_instantiations_are_the_known_variants(so_path):
    found = compiled_variants(so_path)
    assert len(wv.ALL_VARIANTS) == 19
    assert found == wv.ALL_VARIANTS, ("not in ALL_VARIANTS: %s; not compiled: %s"
                                      % (sorted(found - wv.ALL_VARIANTS), sorted(wv.ALL_VARIANTS - found)))


@pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None,
                    reason="needs cuobjdump and cu++filt from the CUDA toolkit")
def test_compiled_ctc_instantiations_are_the_known_variants(so_path):
    """csrc/ctc2d.cu: every compiled ctc2d_* / ctc1d_* / rows_log_softmax kernel is reachable or listed as unreachable"""
    found = {n for n in map(cv.ctc_normalise, compiled_kernels(so_path))
             if re.fullmatch(r"(ctc2d_(?!head)\w+|ctc1d_\w+|rows_log_softmax)_kernel(<[\w,]+>)?", n)}
    assert len(cv.ALL_CTC_VARIANTS) == 70 and len(cv.UNREACHABLE) == 12
    assert found == cv.CTC_KERNELS, ("unknown: %s; not compiled: %s"
                                     % (sorted(found - cv.CTC_KERNELS), sorted(cv.CTC_KERNELS - found)))


def test_every_ctc_variant_has_a_gpu_case():
    covered = test_ctc_variants_gpu.VARIANTS
    assert covered <= cv.ALL_CTC_VARIANTS, sorted(covered - cv.ALL_CTC_VARIANTS)
    assert covered == cv.ALL_CTC_VARIANTS, "no GPU case expects %s" % sorted(cv.ALL_CTC_VARIANTS - covered)


def test_ctc_dispatch_restatement():
    """spot checks of tests/ctc_variants.py against the host dispatch of csrc/ctc2d.cu (132 SMs, 227 KB opt-in)"""
    lim = dict(sms=132, smem=232448)
    p = cv.dp_plan("FAC", 32, 8, 4096, 38, 32, env={}, **lim)
    assert p == {"kernel": "ctc2d_dp4_kernel<1,8>", "family": "dp4", "G": 8}
    assert cv.dp_plan("FAC", 32, 8, 32, 38, 32, env={}, **lim)["G"] == 2              # the grid covers the SMs first
    assert cv.dp_plan("FAC", 32, 8, 4 * 132 + 1, 38, 32, env={}, **lim)["G"] == 4
    assert cv.dp_plan("FAC", 32, 8, 6 * 132 + 1, 38, 32, env={}, **lim)["G"] == 6
    assert cv.dp_plan("GRAD", 48, 8, 8 * 132, 38, 32, env={}, **lim)["G"] == 5         # 75 KB plan shrinks an even G
    assert cv.dp4_pitch(2, 38) == 76 and cv.dp4_pitch(8, 38) == 308
    assert cv.dp_plan("GRAD", 405, 8, 4, 38, 8, env={}, **lim)["family"] == "dp4"
    assert cv.dp_plan("GRAD", 406, 8, 4, 38, 8, env={}, **lim)["kernel"] == "ctc2d_dp_warp_kernel<0,1,8>"
    assert cv.dp_plan("GRAD", 32, 8, 4, 64, 32, env={}, **lim)["family"] == "dp4"
    assert cv.dp_plan("GRAD", 32, 8, 4, 65, 32, env={}, **lim)["kernel"] == "ctc2d_dpg_kernel<0>"
    assert cv.dp_plan("GRAD", 32, 8, 4, 38, 33, env={}, **lim)["kernel"] == "ctc2d_dp_warp_kernel<0,3,8>"
    assert cv.dp_plan("FAC", 32, 2, 4, 38, 16, env={"MR_CTC2D_DP_V3": "1"}, **lim)["kernel"] == \
        "ctc2d_dp_warp_kernel<1,2,0>"
    assert cv.dp_plan("FAC", 32, 8, 4, 38, 16, env={"MR_CTC2D_BLOCK_DP": "1"}, **lim)["kernel"] == \
        "ctc2d_dp_kernel<float,true,1,8>"
    assert cv.dp_plan("FAC_STD", 65, 1, 512, 38, 32, env={}, **lim) == {
        "kernel": "ctc2d_dp_warp_kernel<2,3,0>", "family": "dp_warp", "G": 4, "NSMAX": 3}
    assert cv.dp_plan("FAC_STD", 65, 1, 512, 38, 32, fast=False, env={}, **lim)["kernel"] == "ctc2d_dp_kernel<float,false,2,0>"
    assert cv.dp_plan("GRAD", 16, 8, 4, 38, 32, real="double", env={}, **lim)["kernel"] == "ctc2d_dp_kernel<double,false,0,8>"
    w = cv.dp_plan("GRAD", 12, 8, 4, 38, 256, env={}, **lim)
    assert w["kernel"] == "ctc2d_dp_warp_kernel<0,32,8>" and w["G"] == 4
    assert cv.sample_sweeps(w, 256, [0, 15, 16, 31, 32, 47, 48, 63, 64, 127, 128, 255, 256]) == [
        "warp_sweeps<%d>" % n for n in (1, 1, 2, 2, 3, 3, 4, 4, 8, 8, 16, 16, 32)]
    assert cv.sample_sweeps(p, 32, [0, 15, 16, 31, 32]) == ["warp_sweeps4<%d>" % n for n in (1, 1, 2, 2, 3)]
    assert cv.dp4_rounds(p, 32, [32, 32, 32, 1, 0, 5, 5, 5]) == [2]                     # 3+3+3 slots > 8: a second round
    assert cv.alpha_variant(32, 8, 38, 32, smem=232448) == "ctc2d_alpha_kernel<float,true,true,8>"
    assert cv.alpha_variant(6, 4, 4001, 3, smem=232448) == "ctc2d_alpha_kernel<float,true,false,0>"
    assert cv.alpha_variant(6, 8, 1000, 3, real="double", smem=232448) == "ctc2d_alpha_kernel<double,false,false,0>"
    assert cv.apply_variant(8, 6, 38) == "ctc2d_apply_kernel<true,4,8>"
    assert cv.apply_variant(8, 7, 38) == "ctc2d_apply_kernel<true,1,0>"
    assert cv.apply_variant(3, 4, 7, fast=False, aligned=False) == "ctc2d_apply_kernel<false,1,0>"
    assert cv.ctc_normalise("void <unnamed>::ctc2d_dp_kernel<float, (bool)1, (int)2, (int)0>(<unnamed>::Geo, const T1 *)") \
        == "ctc2d_dp_kernel<float,true,2,0>"
    assert cv.ctc_normalise("<unnamed>::rows_log_softmax_kernel(const float *, long, int, float *)") == "rows_log_softmax_kernel"


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


@pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None,
                    reason="needs cuobjdump and cu++filt from the CUDA toolkit")
def test_compiled_nn_kernels_are_the_known_kernels(so_path):
    """csrc/nn_kernels.cu: every compiled kernel is restated by nn_variants or tested through its own entry elsewhere"""
    from megreader_b200 import build
    found = {nv.nn_normalise(n) for n in compiled_kernels(os.path.join(build.OBJ, "nn_kernels.o"))}
    known = nv.REACHABLE | set(nv.COVERED_ELSEWHERE)
    assert len(nv.REACHABLE) == 56 and len(nv.COVERED_ELSEWHERE) == 7
    assert found == known, "unknown: %s; not compiled: %s" % (sorted(found - known), sorted(known - found))


def test_every_nn_kernel_has_a_gpu_case():
    covered = test_nn_streaming_gpu.KERNELS
    assert covered <= nv.REACHABLE, sorted(covered - nv.REACHABLE)
    assert covered == nv.REACHABLE, "no GPU case expects %s" % sorted(nv.REACHABLE - covered)
    for kernel, test in nv.COVERED_ELSEWHERE.items():
        module, name = test.split("::")
        mod = {"tests/test_decode_gpu.py": test_decode_gpu, "tests/test_nn_kernels_gpu.py": test_nn_kernels_gpu}[module]
        assert callable(getattr(mod, name, None)), "%s: %s is gone" % (kernel, test)


def test_nn_dispatch_restatement():
    """spot checks of tests/nn_variants.py against the host code of csrc/nn_kernels.cu (132 SMs)"""
    P = nv.plan
    # mr_bias_relu_pool_fwd: the row kernel needs a 2x2 window and a power-of-two channel-vector count <= 256
    assert P("mr_bias_relu_pool_fwd", "bf16", 512, 16, 128, 128, (2, 2), (2, 2), (0, 0)) == {"pool_fwd_rows_kernel<bf16,2,2>"}
    assert P("mr_bias_relu_pool_fwd", "float", 2, 8, 8, 24, (2, 2), (2, 2), (0, 0)) == {"bias_relu_pool_fwd_kernel<float>"}
    assert P("mr_bias_relu_pool_fwd", "bf16", 1, 8, 8, 4096, (2, 2), (2, 2), (0, 0)) == {"bias_relu_pool_fwd_kernel<bf16>"}
    # mr_bias_relu_pool_bwd: tiled / hpair / rows / generic, partials for the fused bias gradient
    assert P("mr_bias_relu_pool_bwd", "bf16", 512, 16, 128, 128, (2, 2), (2, 2), (0, 0)) == {
        "pool_bwd_tiled_rows_kernel<bf16,2,2>", "partials_finalize_kernel", "sums_to_float_kernel"}
    assert "pool_bwd_hpair_rows_kernel<bf16,2>" in P("mr_bias_relu_pool_bwd", "bf16", 512, 8, 64, 256, (2, 2), (2, 1), (0, 1))
    assert "pool_bwd_hpair_rows_kernel<bf16,2>" in P("mr_bias_relu_pool_bwd", "bf16", 512, 4, 65, 512, (2, 2), (2, 1), (0, 1))
    assert "pool_bwd_rows_kernel<float,2,2>" in P("mr_bias_relu_pool_bwd", "float", 1, 9, 9, 64, (2, 2), (1, 1), (0, 0))
    assert "pool_bwd_rows_kernel<float,2,2>" in P("mr_bias_relu_pool_bwd", "float", 1, 5, 8, 64, (2, 2), (2, 2), (0, 0))
    assert P("mr_bias_relu_pool_bwd", "float", 2, 9, 9, 64, (3, 3), (3, 3), (0, 0), want_dbias=False) == {
        "bias_relu_pool_bwd_tiled_kernel<float>"}
    assert P("mr_bias_relu_pool_bwd", "float", 2, 8, 8, 24, (2, 2), (2, 2), (0, 0)) == {
        "bias_relu_pool_bwd_tiled_kernel<float>", "col_reduce_kernel<float,2>", "partials_finalize_kernel",
        "sums_to_float_kernel"}                                 # 256 % 6 != 0: the bias gradient is a column sum
    assert nv.pool_bwd("bf16", 2, 8, 8, 64, (2, 2), (2, 2), (0, 0), scratch=False)[0] == {
        "bias_relu_pool_bwd_tiled_kernel<bf16>", "sums_to_float_kernel"}       # fp64 atomics: allocation failed only
    # launch_reduce: partials unless 2C > 4096
    assert nv.reduce_plan(0, "float", 262144, 256)[1] == "partials"
    assert nv.reduce_plan(0, "bf16", 4096, 2048)[1] == "partials"
    assert nv.reduce_plan(0, "bf16", 4096, 2056)[1] == "atomics"
    assert nv.reduce_plan(2, "float", 10 ** 9, 4)[1] == "partials"
    # BatchNorm: row kernels iff the channel-vector count divides 256
    assert P("mr_bn_train_fwd", "bf16", 262144, 256) == {"col_reduce_kernel<bf16,0>", "partials_finalize_kernel",
                                                          "bn_finalize_kernel<bf16>", "bn_apply_rows_kernel<bf16>"}
    assert "bn_apply_kernel<float>" in P("mr_bn_train_fwd", "float", 100, 24)
    assert nv.bn_train_bwd("float", 262144, 24)[2] == "partials" and \
        "bn_bwd_apply_kernel<float>" in P("mr_bn_train_bwd", "float", 262144, 24)
    assert nv.bn_train_bwd("bf16", 4096, 2056)[1:] == ("atomics", "atomics")
    assert nv.bn_bwd_apply_branches("float", 262144, 24) == {"two", "single"}
    assert nv.bn_bwd_apply_branches("bf16", 262144, 40) == {"differs", "single"}
    assert nv.bn_bwd_apply_branches("float", 1000, 24) == {"single"}
    with pytest.raises(nv.Unsupported):
        nv.bn_apply("float", 10, 6)
    # small entries
    assert P("mr_colsum", "float", 500, 38) == {"colsum_scalar_kernel<float>", "sums_to_float_kernel"}
    assert P("mr_bias_act", "bf16", 10, 38) == {"bias_act_scalar_kernel<bf16>"}
    assert P("mr_im2col_nhwc", "float", 3, 27) == {"im2col_scalar_kernel<float>"}
    assert P("mr_im2col_nhwc", "float", 8, 74) == {"im2col_scalar_kernel<float>"}           # Kp % 4 != 0
    with pytest.raises(nv.Unsupported):
        nv.col2im("bf16", 3, 32)
    assert nv.nn_normalise("void (anonymous namespace)::cast_kernel<float, __nv_bfloat16>(float const*, long, "
                           "__nv_bfloat16*)") == "cast_kernel<float,bf16>"
    assert nv.nn_normalise("void <unnamed>::pool_bwd_tiled_rows_kernel<__nv_bfloat16, (int)2, (int)2>(<unnamed>::PoolGeo)") \
        == "pool_bwd_tiled_rows_kernel<bf16,2,2>"
    assert nv.nn_normalise("<unnamed>::partials_finalize_kernel(const float *, int, int, double *)") == \
        "partials_finalize_kernel"
