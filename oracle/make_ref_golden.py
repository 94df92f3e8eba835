"""Record what the reference's OWN CUDA kernels (oracle/_ref/*.so, oracle/build_ref.py) return for every case of
tests/test_ref_kernels_gpu.py into tests/golden/refk_<op>.npz, so that the comparison runs where the reference is absent.

    python -m oracle.make_ref_golden            # needs a GPU and the built oracle/_ref

The test module itself drives the reference kernels (its _references hook); this script only collects what they returned,
cut down by tests.cases.sample_indices to a fixed seeded sample per array (stored with its flat indices, "<key>__idx").
"""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main(out_dir=None):
    import torch
    from oracle import build_ref
    from tests import test_ref_kernels_gpu as T
    from tests.cases import sample_indices
    out_dir = out_dir or T.GOLD
    os.makedirs(out_dir, exist_ok=True)
    store = {}

    def record(op, case_id, names, run_live, share=None):
        mod = build_ref.load("ref_" + op)
        assert mod is not None, "oracle/_ref/ref_%s.so is not built" % op
        live = run_live(mod)
        torch.cuda.synchronize()
        flat = {n: t.cpu().numpy().reshape(-1) for n, t in zip(names, live)}
        for n, a in flat.items():
            idx = sample_indices(flat[(share or {}).get(n, n)])
            store.setdefault(op, {})["%s.%s" % (case_id, n)] = a.copy() if idx is None else a[idx]
            if idx is not None:
                store[op]["%s.%s__idx" % (case_id, n)] = idx.astype(np.int32 if a.size < (1 << 31) else np.int64)
        raise pytest.skip.Exception("recorded")
    T._references = record
    cuda = torch.device("cuda:0")

    def run(fn, *a):
        try:
            fn(cuda, *a)
        except pytest.skip.Exception:
            pass
    for case in T.CTC_CASES:
        for dt in (np.float32, np.float64):
            run(T.test_ctc2d_vs_reference_kernels, case, dt)
    for case in T.DCN_CASES:
        run(T.test_dcnv2_vs_reference_kernels, case)
    for case in T.DCNV1_CASES:
        run(T.test_dcnv1_vs_reference_kernels, case)
    for name in sorted(T.POOL_CASES):
        run(T.test_deform_pool_vs_reference_kernels, name)
    for op, arrays in store.items():
        np.savez_compressed(os.path.join(out_dir, "refk_%s.npz" % op), **arrays)
        print(op, len(arrays), "arrays")


if __name__ == "__main__":
    main(*sys.argv[1:2])
