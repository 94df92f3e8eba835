"""ORACLE — TEST INFRASTRUCTURE ONLY.  CPU restatement ("port") of the reference's CRNN recognition path in plain
PyTorch, used (a) as the parity checker where the reference tree is absent and (b) as the CPU arm of
bench.py (`--impl reference`, `cpu_baseline`).  It is validated bit-for-bit against the UNMODIFIED reference
modules by tests/test_oracle_crnn.py.

  CRNNBackbonePort  <- backbones/crnn.py:4-63   (7 conv blocks; BN blocks have no ReLU, :51-54)
  BiLSTMPort        <- decoders/crnn.py:8-24
  CRNNDecoderPort   <- decoders/crnn.py:27-104  (train: log_softmax -> float64 -> nn.CTCLoss(zero_infinity=True), :95-99)
"""
import torch
import torch.nn as nn


class CRNNBackbonePort(nn.Module):
    def __init__(self, imgH=32, nc=3):
        super().__init__()
        ks, ps, ch = [3, 3, 3, 3, 3, 3, 2], [1, 1, 1, 1, 1, 1, 0], [64, 128, 256, 256, 512, 512, 512]

        def layer(i, bn=False):
            cin = nc if i == 0 else ch[i - 1]
            mods = [nn.Conv2d(cin, ch[i], ks[i], 1, ps[i])]
            mods.append(nn.BatchNorm2d(ch[i]) if bn else nn.ReLU())
            return nn.Sequential(*mods)
        self.cnn = nn.Sequential(
            nn.Sequential(layer(0), nn.MaxPool2d((2, 2))),
            nn.Sequential(layer(1), nn.MaxPool2d((2, 2))),
            layer(2, True),
            nn.Sequential(layer(3), nn.MaxPool2d((2, 2), (2, 1), (0, 1))),
            layer(4, True),
            nn.Sequential(layer(5), nn.MaxPool2d((2, 2), (2, 1), (0, 1))),
            layer(6, True))

    def forward(self, x):
        return self.cnn(x)


class BiLSTMPort(nn.Module):
    def __init__(self, nIn, nHidden, nOut):
        super().__init__()
        self.rnn = nn.LSTM(nIn, nHidden, bidirectional=True)
        self.embedding = nn.Linear(nHidden * 2, nOut)

    def forward(self, x):
        rec, _ = self.rnn(x)
        T, b, h = rec.size()
        return self.embedding(rec.view(T * b, h)).view(T, b, -1)


class CRNNDecoderPort(nn.Module):
    def __init__(self, n_classes=38, inner_channels=256, in_channels=512):
        super().__init__()
        self.rnn = nn.Sequential(BiLSTMPort(in_channels, inner_channels, inner_channels),
                                 BiLSTMPort(inner_channels, inner_channels, n_classes))
        self.ctc_loss = nn.CTCLoss(zero_infinity=True)

    def forward(self, feature, targets=None, lengths=None, train=False):
        b, c, h, w = feature.size()
        assert h == 1
        pred = self.rnn(feature.squeeze(2).permute(2, 0, 1))
        if train:
            pred = nn.functional.log_softmax(pred, dim=2).to(torch.float64)
            pred_size = torch.Tensor([pred.size(0)] * b).int()
            return self.ctc_loss(pred, targets, pred_size, lengths), pred
        return nn.functional.softmax(pred.permute(1, 2, 0).unsqueeze(2), dim=1)


def greedy_ctc_decode(prob, blank=0, unknown=1):
    """structure/representers/ctc_representer.py:22-34: argmax over C, collapse repeats, skip `unknown` without
    updating `previous`, drop blanks.  prob (N, C, 1, W) -> int32 (N, W) blank-padded."""
    pred = torch.argmax(prob, dim=1).select(1, 0)
    out = torch.zeros(pred.shape[0], pred.shape[-1], dtype=torch.int32) + blank
    for i in range(pred.shape[0]):
        valid, previous = 0, blank
        for j in range(pred.shape[1]):
            c = int(pred[i][j])
            if c == previous or c == unknown:
                continue
            if c != blank:
                out[i][valid] = c
                valid += 1
            previous = c
    return out
