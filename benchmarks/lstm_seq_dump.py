"""Outputs of the persistent BiLSTM recurrence kernels on seeded inputs, for comparing two builds bit for bit.
    python benchmarks/lstm_seq_dump.py OUT_DIR             # writes OUT_DIR/lstm_seq_T{T}_N{N}_H{H}.pt per shape
    python benchmarks/lstm_seq_dump.py --compare DIR_A DIR_B
Per shape (T, N, H): the activated gates G, cell states C and layer output Y of mr_lstm_seq_fwd_tcgen05, and the gate
gradients dG of mr_lstm_seq_bwd_tcgen05 on that G and C.  Inputs come from a CPU generator, so every build sees the same
bits.  A shape whose persistent launch is refused, or whose error word is set, fails the run."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

SHAPES = [(65, 512, 256), (26, 300, 256), (5, 100, 128)]


def dump(T, N, H, dev):
    from megreader_b200 import nnops as ops
    g = torch.Generator().manual_seed(1000 * T + N + H)
    Whh = [(torch.randn(4 * H, H, generator=g) / H ** 0.5).bfloat16().to(dev) for _ in range(2)]
    bias = [(torch.randn(4 * H, generator=g) * 0.1).to(dev) for _ in range(2)]
    G = torch.randn(2, T, N, 4 * H, generator=g).bfloat16().to(dev)
    dY = torch.randn(T, N, 2 * H, generator=g).bfloat16().to(dev)
    C = torch.empty(2, T, N, H, device=dev)
    Y = torch.empty(T, N, 2 * H, device=dev, dtype=torch.bfloat16)
    dG = torch.empty_like(G)
    flags = ops.lstm_seq_flags(N, dev)
    assert ops.lstm_seq_fwd_tc(Whh, G, bias, C, Y, flags), "persistent forward refused"
    torch.cuda.synchronize()
    assert int(flags[-1]) == 0, "forward error word %d" % int(flags[-1])
    WhhT = [w.t().contiguous() for w in Whh]
    assert ops.lstm_seq_bwd_tc(WhhT, G, C, dY, dG, flags), "persistent backward refused"
    torch.cuda.synchronize()
    assert int(flags[-1]) == 0, "backward error word %d" % int(flags[-1])
    return {"G": G.cpu(), "C": C.cpu(), "Y": Y.cpu(), "dG": dG.cpu()}


def name(T, N, H):
    return "lstm_seq_T%d_N%d_H%d.pt" % (T, N, H)


def main():
    if sys.argv[1] == "--compare":
        a, b = sys.argv[2], sys.argv[3]
        ok = True
        for shape in SHAPES:
            x, y = torch.load(os.path.join(a, name(*shape))), torch.load(os.path.join(b, name(*shape)))
            for k in ("G", "C", "Y", "dG"):
                same = torch.equal(x[k], y[k])
                ok &= same
                diff = 0.0 if same else float((x[k].float() - y[k].float()).abs().max())
                print("T=%d N=%d H=%d %-2s equal=%s max_abs_diff=%g" % (*shape, k, same, diff))
        print("ALL_EQUAL" if ok else "DIFFERENT")
        sys.exit(0 if ok else 1)
    out = sys.argv[1]
    os.makedirs(out, exist_ok=True)
    dev = torch.device("cuda:0")
    for shape in SHAPES:
        torch.save(dump(*shape, dev), os.path.join(out, name(*shape)))
        print("wrote", name(*shape), flush=True)


if __name__ == "__main__":
    main()
