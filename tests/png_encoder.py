"""A PNG writer in numpy over stdlib zlib, for the decoder tests: every colour type and bit depth, a filter chosen per row
(all five), Adam7 (with empty passes for images under 8 pixels a side), IDAT split at arbitrary points (zero-length chunks
too), any compressobj level / strategy / wbits, ancillary chunks (tEXt, gAMA, eXIf in either byte order, before or after
IDAT), the two APNG orders, and a deflate bit-writer for streams zlib does not emit (a one-code distance tree, a block
without distances, stored blocks of 0 and 65,535 bytes, 258-byte matches at distance 32,768) and broken ones."""
import struct
import zlib

import numpy as np

SIG = b"\x89PNG\r\n\x1a\n"
CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}
DEPTHS = {0: (1, 2, 4, 8, 16), 2: (8, 16), 3: (1, 2, 4, 8), 4: (8, 16), 6: (8, 16)}
ADAM7 = [(0, 0, 8, 8), (4, 0, 8, 8), (0, 4, 4, 8), (2, 0, 4, 4), (0, 2, 2, 4), (1, 0, 2, 2), (0, 1, 1, 2)]


def chunk(ty, data, crc=None):
    c = zlib.crc32(ty + data) if crc is None else crc
    return struct.pack(">I", len(data)) + ty + data + struct.pack(">I", c & 0xFFFFFFFF)


def exif_tiff(orientation, big_endian=False):
    """TIFF data with IFD0 orientation: the payload of a PNG eXIf chunk"""
    e = ">" if big_endian else "<"
    head = (b"MM" if big_endian else b"II") + struct.pack(e + "HI", 42, 8)
    return head + struct.pack(e + "H", 1) + struct.pack(e + "HHIH", 0x0112, 3, 1, orientation) + b"\0\0" + struct.pack(e + "I", 0)


def _pack_row(samples, depth):
    """one row of samples (uint) -> bytes"""
    if depth == 16:
        return samples.astype(">u2").tobytes()
    if depth == 8:
        return samples.astype(np.uint8).tobytes()
    per = 8 // depth
    s = samples.astype(np.uint16)
    pad = (-len(s)) % per
    s = np.concatenate([s, np.zeros(pad, np.uint16)]).reshape(-1, per)
    shifts = (8 - depth * (np.arange(per) + 1)).astype(np.uint16)
    return (s << shifts).sum(1).astype(np.uint8).tobytes()


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))


def _filter(row, prev, ftype, bpp):
    x = np.frombuffer(row, np.uint8).astype(np.int32)
    b = np.frombuffer(prev, np.uint8).astype(np.int32) if prev is not None else np.zeros_like(x)
    a = np.concatenate([np.zeros(bpp, np.int32), x[:-bpp]])[:len(x)]
    c = np.concatenate([np.zeros(bpp, np.int32), b[:-bpp]])[:len(x)]
    pred = [np.zeros_like(x), a, b, (a + b) >> 1, _paeth(a, b, c)][ftype]
    return bytes([ftype]) + ((x - pred) & 255).astype(np.uint8).tobytes()


def raw_data(samples, ctype, depth, interlace=False, filters=None, rng=None):
    """the filtered scanlines of samples (h, w, channels) as bytes; filters: None (all five in turn), an int, or 'random'"""
    h, w = samples.shape[:2]
    bits = CHANNELS[ctype] * depth
    bpp = max(1, bits // 8)
    passes = ADAM7 if interlace else [(0, 0, 1, 1)]
    out, k = bytearray(), 0
    for x0, y0, dx, dy in passes:
        sub = samples[y0::dy, x0::dx]
        if sub.shape[0] == 0 or sub.shape[1] == 0:
            continue
        prev = None
        for r in range(sub.shape[0]):
            row = _pack_row(sub[r].reshape(-1), depth)
            if filters is None:
                f = k % 5
            elif filters == "random":
                f = int(rng.integers(0, 5))
            else:
                f = int(filters)
            out += _filter(row, prev, f, bpp)
            prev = row
            k += 1
    return bytes(out)


def compress(raw, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, wbits=15):
    c = zlib.compressobj(level, zlib.DEFLATED, wbits, 8, strategy)
    return c.compress(raw) + c.flush()


def split(z, cuts):
    """IDAT payloads cut at the given positions (repeats give zero-length chunks)"""
    cuts = [0] + sorted(min(max(int(c), 0), len(z)) for c in cuts) + [len(z)]
    return [z[a:b] for a, b in zip(cuts[:-1], cuts[1:])]


def encode(samples, ctype, depth, interlace=False, filters=None, rng=None, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, wbits=15,
           cuts=(), palette=None, trns=None, before=(), after=(), zdata=None, ihdr=None):
    """a PNG file.  samples: (h, w, channels) unsigned ints of the bit depth; palette: (n, 3) uint8 for colour type 3;
    before / after: extra chunks (bytes) before the first IDAT / after the last; zdata replaces the zlib stream"""
    samples = np.asarray(samples)
    if samples.ndim == 2:
        samples = samples[:, :, None]
    h, w = samples.shape[:2]
    head = ihdr if ihdr is not None else struct.pack(">IIBBBBB", w, h, depth, ctype, 0, 0, int(interlace))
    out = SIG + chunk(b"IHDR", head)
    if palette is not None:
        out += chunk(b"PLTE", np.asarray(palette, np.uint8).tobytes())
    if trns is not None:
        out += chunk(b"tRNS", trns)
    for c in before:
        out += c
    z = zdata if zdata is not None else compress(raw_data(samples, ctype, depth, interlace, filters, rng), level, strategy, wbits)
    for part in split(z, cuts):
        out += chunk(b"IDAT", part)
    for c in after:
        out += c
    return out + chunk(b"IEND", b"")


def random_samples(rng, h, w, ctype, depth, smooth=True):
    c = CHANNELS[ctype]
    hi = (1 << depth) - 1
    if smooth and depth >= 8:
        y, x = np.mgrid[0:h, 0:w]
        base = np.stack([(np.sin(x / rng.uniform(2, 9) + k) * np.cos(y / rng.uniform(2, 9) - k) + 1) / 2 for k in range(c)], -1)
        s = base * hi + rng.normal(0, hi * 0.03, base.shape)
        return np.clip(np.round(s), 0, hi).astype(np.uint32)
    return rng.integers(0, hi + 1, (h, w, c)).astype(np.uint32)


# ---------------------------------------------------------------- APNG

def actl(frames=1):
    return chunk(b"acTL", struct.pack(">II", frames, 0))


def fctl(seq, w, h):
    return chunk(b"fcTL", struct.pack(">IIIIIHHBB", seq, w, h, 0, 0, 1, 10, 0, 0))


def fdat(seq, z):
    return chunk(b"fdAT", struct.pack(">I", seq) + z)


# ---------------------------------------------------------------- deflate bit-writer

class BitWriter:
    def __init__(self):
        self.bits, self.n, self.out = 0, 0, bytearray()

    def put(self, v, k):
        self.bits |= (int(v) & ((1 << k) - 1)) << self.n
        self.n += k
        while self.n >= 8:
            self.out.append(self.bits & 255)
            self.bits >>= 8
            self.n -= 8

    def code(self, c, k):                # Huffman codes go most significant bit first
        r = 0
        for i in range(k):
            r |= ((c >> i) & 1) << (k - 1 - i)
        self.put(r, k)

    def align(self):
        if self.n:
            self.put(0, 8 - self.n)

    def data(self):
        self.align()
        return bytes(self.out)


LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEXT = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DBASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193,
         12289, 16385, 24577]
DEXT = [0, 0, 0, 0] + [k // 2 for k in range(2, 28)]


def canonical(lengths):
    """canonical codes of a length list"""
    maxl = max(lengths) if lengths else 0
    bl = [0] * (maxl + 2)
    for L in lengths:
        if L:
            bl[L] += 1
    code, nxt = 0, [0] * (maxl + 2)
    for b in range(1, maxl + 1):
        code = (code + bl[b - 1]) << 1
        nxt[b] = code
    out = []
    for L in lengths:
        if L:
            out.append(nxt[L])
            nxt[L] += 1
        else:
            out.append(None)
    return out


def fixed_lengths():
    return [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8, [5] * 30


def _len_sym(n):
    for i in range(28, -1, -1):
        if n >= LBASE[i]:
            return i, n - LBASE[i]


def _dist_sym(d):
    for i in range(29, -1, -1):
        if d >= DBASE[i]:
            return i, d - DBASE[i]


def write_tokens(w, tokens, ll, dl):
    """tokens: ints (literals), ('m', length, distance), 'end'; ll / dl: code lengths"""
    lc, dc = canonical(ll), canonical(dl)
    for t in tokens:
        if isinstance(t, tuple):
            _, n, d = t
            s, e = _len_sym(n)
            w.code(lc[257 + s], ll[257 + s])
            w.put(e, LEXT[s])
            s, e = _dist_sym(d)
            w.code(dc[s], dl[s])
            w.put(e, DEXT[s])
        elif t == "end":
            w.code(lc[256], ll[256])
        else:
            w.code(lc[t], ll[t])


def dynamic_header(w, ll, dl, cl_override=None):
    """HLIT / HDIST / HCLEN and the code lengths: runs of zeros as 17 / 18, repeats as 16; cl_override replaces the
    code-length code's lengths (for broken streams)"""
    seq = list(ll) + list(dl)
    syms = []
    i = 0
    while i < len(seq):
        v = seq[i]
        j = i
        while j < len(seq) and seq[j] == v:
            j += 1
        run = j - i
        if v == 0 and run >= 11:
            k = min(run, 138)
            syms.append((18, k - 11))
            i += k
        elif v == 0 and run >= 3:
            syms.append((17, run - 3))
            i += run
        elif v != 0 and run >= 4:
            syms.append((v, None))
            k = min(run - 1, 6)
            syms.append((16, k - 3))
            i += 1 + k
        else:
            syms.append((v, None))
            i += 1
    freq = [0] * 19
    for s, _ in syms:
        freq[s] += 1
    cl = cl_override or _complete([f > 0 for f in freq])
    order = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
    w.put(len(ll) - 257, 5)
    w.put(len(dl) - 1, 5)
    w.put(19 - 4, 4)
    for o in order:
        w.put(cl[o], 3)
    cc = canonical(cl)
    for s, e in syms:
        w.code(cc[s], cl[s])
        if s == 16:
            w.put(e, 2)
        elif s == 17:
            w.put(e, 3)
        elif s == 18:
            w.put(e, 7)


def lengths_for(tokens, nd=30):
    """complete code lengths for the symbols the tokens use (a flat length-9 / length-5 code over them)"""
    ll = [0] * 286
    dl = [0] * nd
    for t in tokens:
        if isinstance(t, tuple):
            ll[257 + _len_sym(t[1])[0]] = 1
            dl[_dist_sym(t[2])[0]] = 1
        elif t == "end":
            ll[256] = 1
        else:
            ll[t] = 1
    return _complete(ll), _complete(dl)


def _complete(used):
    n = sum(1 for u in used if u)
    if n == 0:
        return [0] * len(used)
    if n == 1:
        return [1 if u else 0 for u in used]
    k = max(1, (n - 1).bit_length())
    out, left = [], (1 << k) - n         # give `left` symbols a length one shorter so the code is complete
    for u in used:
        if not u:
            out.append(0)
        elif left > 0:
            out.append(k - 1)
            left -= 1
        else:
            out.append(k)
    # k - 1 lengths: each frees one slot at length k; fix the count so that sum 2^-l == 1
    while sum(2.0 ** -L for L in out if L) > 1:
        i = max(i for i, L in enumerate(out) if L == k - 1)
        out[i] = k
    return out


def zlib_wrap(deflate, data, cinfo=7, adler=None):
    cmf = (cinfo << 4) | 8
    flg = 31 - ((cmf << 8) % 31)
    a = zlib.adler32(data) if adler is None else adler
    return bytes([cmf, flg % 256 if flg != 31 else 0]) + deflate + struct.pack(">I", a & 0xFFFFFFFF)


def tokens_to_bytes(tokens):
    out = bytearray()
    for t in tokens:
        if isinstance(t, tuple):
            for _ in range(t[1]):
                out.append(out[-t[2]])
        elif t != "end":
            out.append(t)
    return bytes(out)


def deflate_dynamic(blocks, final=True):
    """blocks: lists of tokens (each ending in 'end'), one dynamic block each"""
    w = BitWriter()
    for i, toks in enumerate(blocks):
        ll, dl = lengths_for(toks)
        w.put(1 if (final and i == len(blocks) - 1) else 0, 1)
        w.put(2, 2)
        dynamic_header(w, ll, dl)
        write_tokens(w, toks, ll, dl)
    return w.data()


def deflate_stored(chunks):
    w = BitWriter()
    for i, c in enumerate(chunks):
        w.put(1 if i == len(chunks) - 1 else 0, 1)
        w.put(0, 2)
        w.align()
        w.put(len(c), 16)
        w.put(len(c) ^ 0xFFFF, 16)
        for b in c:
            w.put(b, 8)
    return w.data()
