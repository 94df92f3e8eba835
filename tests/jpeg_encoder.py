"""A small numpy baseline JPEG encoder for what neither cv2 nor PIL writes: quantised coefficient blocks given directly
(extreme values that leave 16 bits in the IDCT), 16-bit quantisation tables with large values, Huffman tables with 16-bit
codes, and headers of the processes and component layouts the decoder refuses.

encode(blocks, quant, h, w, ...) writes one interleaved 4:4:4 (or grey) scan of the blocks [ncomp, by, bx, 8, 8] (natural
order) with quantisation tables quant [ncomp, 64] (natural order).  header_only(...) writes the markers of an image whose
frame or scan the decoder refuses, followed by a few entropy-coded bytes and EOI."""
import numpy as np

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14,
                   21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60,
                   61, 54, 47, 55, 62, 63])


def tables(long_codes=False):
    """(DC (bits, vals), AC (bits, vals)) covering every symbol; long_codes gives DC category 0 and EOB 16-bit codes"""
    if long_codes:
        dc = ({5: 15, 16: 1}, list(range(1, 16)) + [0])
        ac = ({8: 254, 9: 1, 16: 1}, list(range(1, 256)) + [0])
    else:
        dc = ({4: 15, 5: 1}, list(range(16)))
        ac = ({8: 255, 9: 1}, list(range(256)))
    return dc, ac


def _codes(spec):
    bits, vals = spec
    code, k, out = 0, 0, {}
    for length in range(1, 17):
        for _ in range(bits.get(length, 0)):
            out[vals[k]] = (code, length)
            code += 1
            k += 1
        code <<= 1
    return out


class _Bits:
    def __init__(self):
        self.out, self.acc, self.n = bytearray(), 0, 0

    def put(self, value, length):
        for i in range(length - 1, -1, -1):
            self.acc = (self.acc << 1) | ((value >> i) & 1)
            self.n += 1
            if self.n == 8:
                self.out.append(self.acc)
                if self.acc == 0xFF:
                    self.out.append(0)
                self.acc, self.n = 0, 0

    def flush(self):
        while self.n:
            self.put(1, 1)
        return bytes(self.out)


def _category(v):
    v = abs(int(v))
    return v.bit_length()


def _extra(v, s):
    return int(v) if v >= 0 else int(v) + (1 << s) - 1


def _segment(marker, payload):
    return bytes([0xFF, marker]) + (len(payload) + 2).to_bytes(2, "big") + payload


def _dqt(quant, sixteen):
    out = b""
    for t, q in enumerate(quant):
        zz = np.asarray(q)[ZIGZAG]
        out += bytes([(0x10 if sixteen else 0) | t]) + (zz.astype(">u2").tobytes() if sixteen else zz.astype(np.uint8).tobytes())
    return _segment(0xDB, out)


def _dht(dc, ac):
    out = b""
    for tc, (bits, vals) in ((0, dc), (1, ac)):
        out += bytes([tc << 4]) + bytes(bits.get(l, 0) for l in range(1, 17)) + bytes(vals)
    return _segment(0xC4, out)


def _sof(marker, precision, h, w, comps):
    p = bytes([precision]) + h.to_bytes(2, "big") + w.to_bytes(2, "big") + bytes([len(comps)])
    for cid, hs, vs, tq in comps:
        p += bytes([cid, (hs << 4) | vs, tq])
    return _segment(marker, p)


def _sos(ids):
    return _segment(0xDA, bytes([len(ids)]) + b"".join(bytes([c, 0x00]) for c in ids) + bytes([0, 63, 0]))


def encode(blocks, quant, h, w, dqt16=False, long_codes=False, marker=0xC0):
    """blocks int [ncomp, by, bx, 8, 8] quantised (natural order), quant [ncomp, 64]; ncomp 1 (grey) or 3 (YCbCr 4:4:4,
    one table per component)"""
    blocks = np.asarray(blocks)
    ncomp, by, bx = blocks.shape[:3]
    assert by == (h + 7) // 8 and bx == (w + 7) // 8
    dc, ac = tables(long_codes)
    cdc, cac = _codes(dc), _codes(ac)
    bw = _Bits()
    pred = [0] * ncomp
    for y in range(by):
        for x in range(bx):
            for c in range(ncomp):
                z = blocks[c, y, x].reshape(64)[ZIGZAG]
                d = int(z[0]) - pred[c]
                pred[c] = int(z[0])
                s = _category(d)
                bw.put(*cdc[s])
                if s:
                    bw.put(_extra(d, s), s)
                run = 0
                for k in range(1, 64):
                    v = int(z[k])
                    if v == 0:
                        run += 1
                        continue
                    while run > 15:
                        bw.put(*cac[0xF0])
                        run -= 16
                    s = _category(v)
                    bw.put(*cac[(run << 4) | s])
                    bw.put(_extra(v, s), s)
                    run = 0
                if run:
                    bw.put(*cac[0x00])
    ids = [1, 2, 3][:ncomp]
    head = b"\xff\xd8" + _dqt(quant, dqt16) + _sof(marker, 8, h, w, [(i, 1, 1, t) for t, i in enumerate(ids)]) + _dht(dc, ac)
    return head + _sos(ids) + bw.flush() + b"\xff\xd9"


def header_only(marker=0xC0, precision=8, h=16, w=16, comps=((1, 1, 1, 0), (2, 1, 1, 0), (3, 1, 1, 0)), scan_ids=None):
    """markers of a frame the decoder refuses (another SOF process, 12-bit samples, height 0, 2 or 4 components,
    fractional sampling, or a scan with fewer components than the frame), a few entropy-coded bytes and EOI"""
    dc, ac = tables()
    q = [np.full(64, 8)]
    ids = scan_ids if scan_ids is not None else [c[0] for c in comps]
    return (b"\xff\xd8" + _dqt(q, False) + _sof(marker, precision, h, w, list(comps)) + _dht(dc, ac) + _sos(ids)
            + bytes([0x12, 0x34, 0x56, 0x78]) + b"\xff\xd9")
