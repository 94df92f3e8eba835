"""Which CTC kernel instantiation a call launches, restated from the host dispatch of csrc/ctc2d.cu.

launch_alpha, launch_dp (with launch_dp4, launch_dpg, launch_dp_warp) and mr_ctc2d_backward_apply_f32 pick one of the
compiled instantiations from the dtype, the fast-math switch, the mode (GRAD: contract backward, FAC: 2D training
forward, FAC_STD: the 1D loss), H == 8, the shared-memory plans (S, C, T), N against the SM count, the 16-byte alignment
of the operands, and the environment switches MR_CTC2D_BLOCK_DP / MR_CTC2D_DP_V3 (read on every call).  Inside the warp
kernels every sample then picks its own sweep width from its target length.

tests/test_ctc_variants_gpu.py asserts through wgmma_variants.launched_kernels() that the expected instantiations ran;
tests/test_kernel_inventory.py checks on the CPU that the compiled instantiations are exactly
ALL_CTC_VARIANTS | UNREACHABLE and that each reachable one is expected by at least one GPU case.

The SM count and the shared-memory opt-in limit are read from the device, as the C++ does, so a case built from
N = k * SMs selects the same group size on any H100.
"""
import os
import warnings

from tests.wgmma_variants import launched_kernels, normalise

MODES = {"GRAD": 0, "FAC": 1, "FAC_STD": 2}
_NS = (1, 2, 3, 4, 8, 16, 32)


def _b(v):
    return "true" if v else "false"


def _cdiv(a, b):
    return -(-a // b)


def ctc_normalise(name):
    """wgmma_variants.normalise, with cu++filt's (bool)0 / (bool)1 spelled as the profiler spells them."""
    return normalise(name.replace("(bool)0", "false").replace("(bool)1", "true"))


# ---------------------------------------------------------------- every compiled instantiation
def _all_compiled():
    out = set()
    for f in (True, False):
        out |= {"ctc2d_alpha_kernel<float,%s,true,8>" % _b(f), "ctc2d_alpha_kernel<float,%s,true,0>" % _b(f),
                "ctc2d_alpha_kernel<float,%s,false,0>" % _b(f)}
        out |= {"ctc2d_dp_kernel<float,%s,%d,%d>" % (_b(f), m, ht) for m in (0, 1, 2) for ht in (8, 0)}
        out |= {"ctc2d_apply_kernel<%s,4,8>" % _b(f), "ctc2d_apply_kernel<%s,4,0>" % _b(f),
                "ctc2d_apply_kernel<%s,1,0>" % _b(f)}
    out |= {"ctc2d_alpha_kernel<double,false,true,8>", "ctc2d_alpha_kernel<double,false,true,0>",
            "ctc2d_alpha_kernel<double,false,false,0>"}
    out |= {"ctc2d_dp_kernel<double,false,0,%d>" % ht for ht in (8, 0)}
    out |= {"ctc2d_dp4_kernel<%d,%d>" % (m, ht) for m in (0, 1, 2) for ht in (8, 0)}
    out |= {"ctc2d_dpg_kernel<%d>" % m for m in (0, 1, 2)}
    out |= {"ctc2d_dp_warp_kernel<%d,%d,%d>" % (m, ns, ht) for m in (0, 1, 2) for ns in _NS for ht in (8, 0)}
    return out | {"rows_log_softmax_kernel", "ctc1d_grad_rows_kernel"}


_H1 = "the 1D loss always has H = 1"
UNREACHABLE = {
    "ctc2d_dp_kernel<float,true,2,8>": _H1,
    "ctc2d_dp_kernel<float,false,2,8>": _H1,
    "ctc2d_dp4_kernel<2,8>": "launch_dp4 refuses MODE_FAC_STD before it launches",
    "ctc2d_dp4_kernel<2,0>": "launch_dp4 refuses MODE_FAC_STD before it launches",
    "ctc2d_dpg_kernel<2>": "launch_dpg refuses MODE_FAC_STD before it launches",
}
UNREACHABLE.update({"ctc2d_dp_warp_kernel<2,%d,8>" % ns: _H1 for ns in _NS})
ALL_CTC_VARIANTS = frozenset(_all_compiled() - set(UNREACHABLE))
CTC_KERNELS = ALL_CTC_VARIANTS | frozenset(UNREACHABLE)


def device_limits():
    """(SM count, shared-memory opt-in bytes per block) of cuda:0, the two numbers the plans read.  Without a device (the
    CPU inventory) those of an H100 SXM: 132 SMs, 227 KB."""
    import torch
    if not torch.cuda.is_available():
        return 132, 232448
    p = torch.cuda.get_device_properties(0)
    return p.multi_processor_count, p.shared_memory_per_block_optin


# ---------------------------------------------------------------- the host dispatch, restated
def alpha_variant(T, H, C, S, real="float", fast=True, smem=None):
    """launch_alpha: the cp.async-staged kernel whenever a group of >= 1 samples fits (<= 56 KB, or the opt-in limit for one
    sample), H = 8 unrolled on that path only; otherwise the unstaged kernel."""
    smem = device_limits()[1] if smem is None else smem
    size = 8 if real == "double" else 4
    SS = 2 * S + 1
    G = min(8, max(1, 288 // SS))
    staged = False
    for g in range(G, 0, -1):
        need = size * 4 * H * g * C + size * (g * C + g * SS + 2 * g)
        if need <= 56 * 1024 or (g == 1 and need <= smem):
            staged = True
            break
    if not staged:
        small = lambda g: size * (g * C + g * SS + 2 * g)  # noqa: E731
        while G > 1 and small(G) > smem:
            G -= 1
        if small(G) > smem:
            raise ValueError("launch_alpha returns MR_ERR_UNSUPPORTED")
    return "ctc2d_alpha_kernel<%s,%s,%s,%d>" % (real, _b(fast and real == "float"), _b(staged),
                                                8 if staged and H == 8 else 0)


def dp4_pitch(G, C):
    """Row pitch of dp4's Q / sum rows: the first value >= G * C that is 4 (mod 8)."""
    return G * C + (4 - G * C) % 8


def dp_plan(mode, T, H, N, C, S, real="float", fast=True, env=None, sms=None, smem=None):
    """launch_dp -> {"kernel": instantiation, "family": dp4 | dpg | dp_warp | dp, "G": samples per CTA (per warp group
    for dpg), "NSMAX": (dp_warp) the launch's states-per-lane}."""
    env = os.environ if env is None else env
    if sms is None or smem is None:
        d_sms, d_smem = device_limits()
        sms = d_sms if sms is None else sms
        smem = d_smem if smem is None else smem
    m, SS, ht = MODES[mode], 2 * S + 1, 8 if H == 8 else 0
    fast = fast and real == "float"
    if fast and mode != "FAC_STD" and "MR_CTC2D_BLOCK_DP" not in env and "MR_CTC2D_DP_V3" not in env:
        if S <= 32 and C <= 64:
            need = lambda g: 4 * (T * dp4_pitch(g, C) + max(g, 3) * T * 33) + 4 * (7 * g + 1 + 64 * g) + 16  # noqa: E731
            G = 8
            while G > 2 and _cdiv(N, G) < sms:
                G -= 2
            while G > 1 and need(G) > 75 * 1024:
                G -= 1
            if need(G) <= smem:
                return {"kernel": "ctc2d_dp4_kernel<%d,%d>" % (m, ht), "family": "dp4", "G": G}
        if C > 64 and S <= 32 and 16 * (T * 132 + 96) <= smem:
            return {"kernel": "ctc2d_dpg_kernel<%d>" % m, "family": "dpg", "G": 4}
    if fast and "MR_CTC2D_BLOCK_DP" not in env:
        ns = min(o for o in _NS if o >= _cdiv(SS, 32))
        need = lambda g: 4 * (T * g * C + g * T * SS + g) + 4 * g * T * _cdiv(C, 32) + 16  # noqa: E731
        G = 8
        while G > 1 and need(G) > 110 * 1024:
            G -= 1
        if need(G) <= smem:
            return {"kernel": "ctc2d_dp_warp_kernel<%d,%d,%d>" % (m, ns, ht), "family": "dp_warp", "G": G, "NSMAX": ns}
    size = 8 if real == "double" else 4
    G = min(8, max(1, 160 // SS))
    need = lambda g: size * (2 * T * g * C + T * g * SS + 2 * g * SS + 3 * g) + T * g * C + 16  # noqa: E731
    while G > 1 and need(G) > 44 * 1024:
        G -= 1
    if need(G) > smem:
        raise ValueError("launch_dp returns MR_ERR_UNSUPPORTED")
    return {"kernel": "ctc2d_dp_kernel<%s,%s,%d,%d>" % (real, _b(fast), m, ht), "family": "dp", "G": G}


def sample_sweeps(plan, S, target_lengths):
    """Per sample, the sweep its warp runs: warp_sweeps<NS> (dp_warp: the smallest of 1, 2, 3, 4, 8, 16, NSMAX that holds
    min(2L+1, 2S+1) states), warp_sweeps4<ns> (dp4 / dpg: ns = ceil((2L+1) / 32), L clamped to S), or None (block kernel)."""
    out = []
    for L in target_lengths:
        L = int(L)
        if plan["family"] == "dp_warp":
            need = _cdiv(min(max(2 * L + 1, 1), 2 * S + 1), 32)
            out.append("warp_sweeps<%d>" % min(o for o in _NS if o >= need and o <= plan["NSMAX"]))
        elif plan["family"] in ("dp4", "dpg"):
            out.append("warp_sweeps4<%d>" % min(3, _cdiv(2 * min(max(L, 0), S) + 1, 32)))
        else:
            out.append(None)
    return out


def dp4_rounds(plan, S, target_lengths):
    """dp4's slot plan: for each CTA, how many rounds its warps run (a sample takes ns slots out of max(G, 3))."""
    G = plan["G"]
    nslots = max(G, 3)
    rounds = []
    for b0 in range(0, len(target_lengths), G):
        used, r = 0, 0
        for L in target_lengths[b0:b0 + G]:
            ns = _cdiv(2 * min(max(int(L), 0), S) + 1, 32)
            if used + ns > nslots:
                r, used = r + 1, 0
            used += ns
        rounds.append(r + 1)
    return rounds


def apply_variant(H, N, C, fast=True, aligned=True):
    """mr_ctc2d_backward_apply_f32: 16-byte vectors when lp, grad and gfac are 16-byte aligned and N*C % 4 == 0; H = 8
    unrolled on the vector path only."""
    v4 = aligned and (N * C) % 4 == 0
    return "ctc2d_apply_kernel<%s,%d,%d>" % (_b(fast), 4 if v4 else 1, 8 if v4 and H == 8 else 0)


def expected_kernels(entry, T, H, N, C, S, fast=True, real="float", aligned=True, env=None):
    """The library kernels one call of `entry` launches:
    contract: ctc2d_forward + ctc2d_backward;  train: ctc_loss_2d forward + backward (the training pair);
    ctc1d: ctc1d.ctc_loss_from_logits forward + backward (H = 1)."""
    if entry == "contract":
        return {alpha_variant(T, H, C, S, real, fast), dp_plan("GRAD", T, H, N, C, S, real, fast, env)["kernel"]}
    if entry == "train":
        return {dp_plan("FAC", T, H, N, C, S, "float", fast, env)["kernel"], apply_variant(H, N, C, fast, aligned)}
    if entry == "ctc1d":
        return {"rows_log_softmax_kernel", dp_plan("FAC_STD", T, 1, N, C, S, "float", fast, env)["kernel"],
                "ctc1d_grad_rows_kernel"}
    raise KeyError(entry)


def run_expecting(expected, fn):
    """fn() must launch exactly the CTC kernels in `expected`; -> fn's result.  Any CTC kernel outside `expected` always
    fails.  As in wgmma_variants.run_variant, a trace that lacks expected records only warns: the profiler was seen to lose
    some or all of the library's kernel records (about one case per run of the CTC file on its own, a different one each
    time; more often late in a long pytest process), so a missing record says nothing about the dispatch.  A kernel that
    did not run at all leaves its outputs unwritten, which the value checks catch."""
    assert expected <= ALL_CTC_VARIANTS, sorted(expected - ALL_CTC_VARIANTS)
    result, names = launched_kernels(fn)
    seen = {ctc_normalise(n) for n in names} & CTC_KERNELS
    assert seen <= expected, "expected %s to run, the profiler saw %s" % (sorted(expected), sorted(seen))
    if seen != expected:
        warnings.warn("torch.profiler recorded no CTC kernel record for %s: not checked (saw %s)"
                      % (sorted(expected - seen), sorted(names)))
    return result
