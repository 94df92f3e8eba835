"""Which csrc/nn_kernels.cu kernels a call launches, restated from the host code of its C entry points.

The streaming entries pick among their kernels by dtype, channel-vector count (C / VN, VN = 4 fp32 or 8 bf16 elements
per 16-byte vector), window geometry, whether a bias gradient is wanted, and whether a per-channel reduction fits the
library's partial-sum scratch (kMaxPartialBlocks = 132 * 8 row blocks of kMaxPartialCols = 4096 columns) or falls back
to fp64 atomics.  plan() returns, for one call, the set of kernels it launches and how its per-channel sums are
reduced.

tests/test_nn_streaming_gpu.py asserts through wgmma_variants.launched_kernels() that the planned kernels ran (once per
kernel) and checks every output against float64; tests/test_kernel_inventory.py checks on the CPU that the compiled
instantiations of nn_kernels.cu are exactly REACHABLE | COVERED_ELSEWHERE, and that each reachable one is planned by at
least one GPU case.

Not covered: N*H*W >= 2^31 pixels (the row kernels' limit, which sends such a pool to the generic kernels) needs tens of
GB of activations and stays untested.
"""
from tests.wgmma_variants import normalise

TYPES = {"float32": "float", "bfloat16": "bf16"}
VN = {"float": 4, "bf16": 8}
K_MAX_PARTIAL_BLOCKS = 132 * 8
K_MAX_PARTIAL_COLS = 4096
SMS = 132                                      # H100 SXM; the GPU tests pass the device's own count


def nn_normalise(name):
    """wgmma_variants.normalise, with __nv_bfloat16 spelled bf16: "cast_kernel<float,bf16>", "adam_kernel"."""
    return normalise(name).replace("__nv_bfloat16", "bf16")


def _cdiv(a, b):
    return -(-a // b)


def _t(dtype):
    """"float32" / "bfloat16" / a torch dtype -> "float" / "bf16" """
    return TYPES[str(dtype).replace("torch.", "")]


def pow2_shift(v):
    if v <= 0 or v & (v - 1):
        return -1
    return v.bit_length() - 1


def grid1d(work, block, per_sm=16, sms=SMS):
    return max(1, min(_cdiv(work, block), sms * per_sm))


class Unsupported(ValueError):
    """the entry returns MR_ERR_UNSUPPORTED"""


def _vec_ok(T, C):
    return C % VN[T] == 0


# ---------------------------------------------------------------- shared pieces
def reduce_plan(mode, T, rows, C, sms=SMS):
    """launch_reduce: col_reduce_kernel<T, mode> on a (ceil(cv/32), gy) grid, then partials_finalize_kernel when the
    gy x 2C partials fit the scratch; else fp64 atomics into `sums`.  -> (kernels, "partials" | "atomics")."""
    if not _vec_ok(T, C):
        raise Unsupported("launch_reduce: C % VN != 0")
    gx = _cdiv(C // VN[T], 32)
    gy = max(1, (sms * 8) // gx)
    rpc = max(64, _cdiv(rows, gy))
    gy = _cdiv(rows, rpc)
    if gy <= K_MAX_PARTIAL_BLOCKS and 2 * C <= K_MAX_PARTIAL_COLS:
        return {"col_reduce_kernel<%s,%d>" % (T, mode), "partials_finalize_kernel"}, "partials"
    return {"col_reduce_kernel<%s,%d>" % (T, mode)}, "atomics"


def colsum_plan(T, rows, C, sms=SMS):
    """mr_colsum: the scalar kernel (fp64 atomics) when C % VN != 0, else launch_reduce MODE 2; then sums_to_float."""
    if not _vec_ok(T, C):
        return {"colsum_scalar_kernel<%s>" % T, "sums_to_float_kernel"}, "atomics"
    ks, how = reduce_plan(2, T, rows, C, sms)
    return ks | {"sums_to_float_kernel"}, how


# ---------------------------------------------------------------- the entries
def pool_fwd(T, N, H, W, C, k, s, p):
    if not _vec_ok(T, C):
        raise Unsupported("mr_bias_relu_pool_fwd: C % VN != 0")
    sft = pow2_shift(C // VN[T])
    if tuple(k) == (2, 2) and 0 <= sft <= 8 and N * H * W < 2 ** 31:
        return {"pool_fwd_rows_kernel<%s,2,2>" % T}, None
    return {"bias_relu_pool_fwd_kernel<%s>" % T}, None


def pool_bwd(T, N, H, W, C, k, s, p, want_dbias=True, scratch=True, sms=SMS):
    """mr_bias_relu_pool_bwd.  H, W are the pool's INPUT size.  `scratch` = False restates a failed scratch allocation,
    which no test can arrange (see UNREACHABLE_BRANCHES)."""
    if not _vec_ok(T, C):
        raise Unsupported("mr_bias_relu_pool_bwd: C % VN != 0")
    (kh, kw), (sh, sw), (ph, pw) = k, s, p
    Ho = (H + 2 * ph - kh) // sh + 1
    cv = C // VN[T]
    fuse = want_dbias and 256 % cv == 0
    part = fuse and C <= K_MAX_PARTIAL_COLS and scratch
    tiled = kh == sh and kw == sw and ph == 0 and pw == 0 and H % kh == 0 and W % kw == 0
    sft = pow2_shift(cv)
    if (kh, kw) == (2, 2) and 0 <= sft <= 8 and (part or not want_dbias) and N * H * W < 2 ** 31:
        if tiled:
            ks = {"pool_bwd_tiled_rows_kernel<%s,2,2>" % T}
        elif sh == 2 and ph == 0 and H % 2 == 0 and Ho * 2 == H:
            ks = {"pool_bwd_hpair_rows_kernel<%s,2>" % T}
        else:
            ks = {"pool_bwd_rows_kernel<%s,2,2>" % T}
    elif tiled:
        ks = {"bias_relu_pool_bwd_tiled_kernel<%s>" % T}
    else:
        ks = {"bias_relu_pool_bwd_kernel<%s>" % T}
    how = None
    if part:
        ks.add("partials_finalize_kernel")
        how = "partials"
    elif fuse:
        how = "atomics"
    if want_dbias:
        if fuse:
            ks.add("sums_to_float_kernel")
        else:
            cks, how = colsum_plan(T, N * H * W, C, sms)
            ks |= cks
    return ks, how


def _bn_apply_kernel(T, C):
    return ("bn_apply_rows_kernel<%s>" if 256 % (C // VN[T]) == 0 else "bn_apply_kernel<%s>") % T


def bn_train_fwd(T, rows, C, sms=SMS):
    ks, how = reduce_plan(0, T, rows, C, sms)
    return ks | {"bn_finalize_kernel<%s>" % T, _bn_apply_kernel(T, C)}, how


def bn_apply(T, rows, C):
    if not _vec_ok(T, C):
        raise Unsupported("mr_bn_apply: C % VN != 0")
    return {_bn_apply_kernel(T, C)}, None


def bn_train_bwd(T, rows, C, want_dbias=True, scratch=True, sms=SMS):
    """-> (kernels, reduction of the statistics, reduction of the fused bias gradient or None)"""
    ks, how = reduce_plan(1, T, rows, C, sms)
    ks = ks | {"sums_to_float_kernel"}
    cv = C // VN[T]
    if 256 % cv == 0:
        ks.add("bn_bwd_apply_rows_kernel<%s>" % T)
        if not want_dbias:
            return ks, how, None
        if scratch:                               # C <= 2048 here, so the [grid, C] partials always fit
            return ks | {"partials_finalize_kernel", "sums_to_float_kernel"}, how, "partials"
        cks, bhow = colsum_plan(T, rows, C, sms)
        return ks | cks, how, bhow
    ks.add("bn_bwd_apply_kernel<%s>" % T)
    if not want_dbias:
        return ks, how, None
    cks, bhow = colsum_plan(T, rows, C, sms)        # `fuse` needs 256 % cv == 0: the bias gradient is a column sum
    return ks | cks, how, bhow


def bn_bwd_apply_branches(T, rows, C, sms=SMS):
    """Which per-thread branches bn_bwd_apply_kernel takes (one grid-stride pass handles t and t2 = t + stride):
    "two" (t2 shares t's channel vector), "differs" (t2 in range with another channel vector), "single" (t2 past the end)."""
    cv = C // VN[T]
    total = rows * cv
    stride = grid1d(total, 256, 32, sms) * 256
    out = set()
    if total > stride:                            # t2 % cv == t % cv for every pair exactly when cv divides the stride
        out.add("two" if stride % cv == 0 else "differs")
    if total % (2 * stride):                      # the last, partial 2-stride block has a t whose t2 is past the end
        out.add("single")
    return out


def bias_act(T, rows, C):
    return {("bias_act_kernel<%s>" if _vec_ok(T, C) else "bias_act_scalar_kernel<%s>") % T}, None


def cast(Ti, To):
    return {"cast_kernel<%s,%s>" % (Ti, To)}, None


def im2col(T, C, Kp):
    return {("im2col_vec_kernel<%s>" if _vec_ok(T, C) and _vec_ok(T, Kp) else "im2col_scalar_kernel<%s>") % T}, None


def col2im(T, C, Kp):
    if not (_vec_ok(T, C) and _vec_ok(T, Kp)):
        raise Unsupported("mr_col2im_nhwc: vector path only")
    return {"col2im_vec_kernel<%s>" % T}, None


def nchw_to_nhwc(T):
    return {"nchw_to_nhwc_kernel<%s>" % T}, None


def nhwc_to_nchw(T):
    return {"nhwc_to_nchw_kernel<%s>" % T}, None


def lstm_cell_fwd(T):
    return {"lstm_cell_fwd_kernel<%s>" % T}, None


def lstm_cell_bwd(T):
    return {"lstm_cell_bwd_kernel<%s>" % T}, None


ENTRIES = {
    "mr_bias_relu_pool_fwd": pool_fwd, "mr_bias_relu_pool_bwd": pool_bwd,
    "mr_bn_train_fwd": bn_train_fwd, "mr_bn_apply": bn_apply, "mr_bn_train_bwd": bn_train_bwd,
    "mr_colsum": colsum_plan, "mr_bias_act": bias_act, "mr_cast": cast,
    "mr_im2col_nhwc": im2col, "mr_col2im_nhwc": col2im,
    "mr_nchw_to_nhwc": nchw_to_nhwc, "mr_nhwc_to_nchw": nhwc_to_nchw,
    "mr_lstm_cell_fwd": lstm_cell_fwd, "mr_lstm_cell_bwd": lstm_cell_bwd,
}


def plan(entry, *args, **kw):
    """-> frozenset of the nn_kernels.cu kernels one call of `entry` launches (the dtype arguments as "float" / "bf16")."""
    return frozenset(ENTRIES[entry](*args, **kw)[0])


# ---------------------------------------------------------------- the compiled set
def _reachable():
    out = set()
    for T in ("float", "bf16"):
        out |= {k % T for k in (
            "nchw_to_nhwc_kernel<%s>", "nhwc_to_nchw_kernel<%s>", "im2col_vec_kernel<%s>", "im2col_scalar_kernel<%s>",
            "col2im_vec_kernel<%s>", "bias_relu_pool_fwd_kernel<%s>", "bias_relu_pool_bwd_kernel<%s>",
            "bias_relu_pool_bwd_tiled_kernel<%s>", "pool_fwd_rows_kernel<%s,2,2>", "pool_bwd_rows_kernel<%s,2,2>",
            "pool_bwd_hpair_rows_kernel<%s,2>", "pool_bwd_tiled_rows_kernel<%s,2,2>", "bias_act_kernel<%s>",
            "bias_act_scalar_kernel<%s>", "col_reduce_kernel<%s,0>", "col_reduce_kernel<%s,1>",
            "col_reduce_kernel<%s,2>", "bn_finalize_kernel<%s>", "bn_apply_kernel<%s>", "bn_apply_rows_kernel<%s>",
            "bn_bwd_apply_kernel<%s>", "bn_bwd_apply_rows_kernel<%s>", "colsum_scalar_kernel<%s>",
            "lstm_cell_fwd_kernel<%s>", "lstm_cell_bwd_kernel<%s>")}
        out |= {"cast_kernel<%s,%s>" % (T, To) for To in ("float", "bf16")}
    return out | {"partials_finalize_kernel", "sums_to_float_kernel"}


REACHABLE = frozenset(_reachable())

# compiled in nn_kernels.cu, but tested through their own entries elsewhere
COVERED_ELSEWHERE = {
    "ctc_greedy_decode_kernel": "tests/test_decode_gpu.py::test_ctc_greedy_decode_bit_exact",
    "blank_after_first_blank_kernel": "tests/test_decode_gpu.py::test_blank_after_first_blank",
    "adam_kernel": "tests/test_nn_kernels_gpu.py::test_adam_matches_torch",
    "conv_weight_pack_kernel<float>": "tests/test_nn_kernels_gpu.py::test_weight_pack_kernels",
    "conv_weight_pack_kernel<bf16>": "tests/test_nn_kernels_gpu.py::test_weight_pack_kernels",
    "gate_rows_permute_kernel<float>": "tests/test_nn_kernels_gpu.py::test_weight_pack_kernels",
    "gate_rows_permute_kernel<bf16>": "tests/test_nn_kernels_gpu.py::test_weight_pack_kernels",
}

# Every compiled instantiation is reachable; these code paths inside them are not.
UNREACHABLE_BRANCHES = {
    "mr_bias_relu_pool_bwd: fp64-atomic block_channel_sum in bias_relu_pool_bwd(_tiled)_kernel":
        "`fuse` needs 256 % cv == 0, so C <= 256 * VN <= 2048 and the [blocks, C] partials always fit the scratch; "
        "the atomics run only when the scratch allocation failed",
    "mr_bias_relu_pool_bwd: a 2x2 window with a fused bias gradient and no partials":
        "the same: (part || !dbias) fails only when the scratch allocation failed",
    "mr_bn_train_bwd: bias_sums in bn_bwd_apply_kernel (and the memset before it)":
        "`fuse` needs 256 % cv == 0, which sends the call to bn_bwd_apply_rows_kernel; bn_bwd_apply_kernel is always "
        "passed NULL",
    "mr_bn_train_bwd: mr_colsum after bn_bwd_apply_rows_kernel with a bias gradient":
        "the rows kernel's C <= 2048 partials always fit the scratch; only a failed allocation leaves `part` NULL",
    "launch_reduce: atomics because gy > kMaxPartialBlocks":
        "gy <= SMs * 8 / gx <= 132 * 8 on an H100; only 2C > 4096 (C > 2048) reaches the atomics",
    "mr_col2im_nhwc: a scalar path":
        "there is none: C or Kp not a multiple of VN returns MR_ERR_UNSUPPORTED",
}
