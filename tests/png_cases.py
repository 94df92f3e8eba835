"""Seeded PNG inputs of the decoder tests and the host harness (tests/host_harness/png_core_host.cpp, the product's
png_core.cuh compiled with g++).

corpus() holds the numpy encoder's files (tests/png_encoder.py: every colour type and bit depth, all five filters, Adam7
with empty passes, split IDATs, zlib levels / strategies / window sizes, ancillary chunks, eXIf orientations, APNG, deflate
streams zlib does not emit), cv2.imencode's (IMWRITE_PNG_COMPRESSION, _STRATEGY, _FILTER, _BILEVEL), PIL's (modes P, 1, L,
LA, I;16), and broken files, whose expected status is in EXPECTED_STATUS."""
import ctypes
import io
import os
import shutil
import struct
import subprocess
import zlib

import numpy as np

from tests import png_encoder as E

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "megreader_b200", "csrc")


def _gxx_cmd(extra, out):
    return [shutil.which("g++"), "-std=c++17", "-I" + CSRC, os.path.join(HERE, "host_harness", "png_core_host.cpp"), "-o", out] + extra


def build_harness(tmp):
    if shutil.which("g++") is None:
        return None
    so = os.path.join(str(tmp), "libpng_core_host.so")
    subprocess.check_call(_gxx_cmd(["-O2", "-shared", "-fPIC"], so))
    L = ctypes.CDLL(so)
    P, I64 = ctypes.c_void_p, ctypes.c_int64
    L.host_header.argtypes = [P, I64, P]
    L.host_decode.argtypes = [P, I64, ctypes.c_int, I64, P, P, P]
    return L


def build_sanitized(tmp):
    """the harness as an executable under AddressSanitizer and UBSan, or None where g++ cannot build one"""
    if shutil.which("g++") is None:
        return None
    exe = os.path.join(str(tmp), "png_core_host_asan")
    cmd = _gxx_cmd(["-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-fno-omit-frame-pointer",
                    "-DPNG_HARNESS_MAIN"], exe)
    if subprocess.run(cmd, capture_output=True).returncode != 0:
        return None
    return exe


def header(L, blob):
    b = np.frombuffer(bytes(blob), np.uint8)
    info = np.zeros(8, np.int32)
    L.host_header(b.ctypes.data, b.size, info.ctypes.data)
    return info


def host_decode(L, blob, jump=0):
    """(status, HWC uint8 array or None, pointer-jumping rounds) of the product's routines on one byte string"""
    b = np.frombuffer(bytes(blob), np.uint8)
    info = header(L, blob)
    cap = max(3 * int(info[1]) * int(info[2]), 1)
    out = np.zeros(cap, np.uint8)
    hw = np.zeros(2, np.int32)
    rounds = np.zeros(1, np.int32)
    st = L.host_decode(b.ctypes.data, b.size, jump, cap, out.ctypes.data, hw.ctypes.data, rounds.ctypes.data)
    if st:
        return st, None, int(rounds[0])
    return 0, out[:3 * hw[0] * hw[1]].reshape(hw[0], hw[1], 3), int(rounds[0])


def header_pixels(blob):
    b = bytes(blob)
    if len(b) < 24 or b[:8] != E.SIG:
        return 0
    return int.from_bytes(b[16:20], "big") * int.from_bytes(b[20:24], "big")


def cv2_encode(img, compression=3, strategy=None, filt=None, bilevel=False):
    import cv2
    p = [cv2.IMWRITE_PNG_COMPRESSION, int(compression)]
    if strategy is not None:
        p += [cv2.IMWRITE_PNG_STRATEGY, int(strategy)]
    if filt is not None:
        p += [cv2.IMWRITE_PNG_FILTER, int(filt)]
    if bilevel:
        p += [cv2.IMWRITE_PNG_BILEVEL, 1]
    ok, b = cv2.imencode(".png", img, p)
    assert ok
    return b.tobytes()


def pil_encode(arr, mode, **kw):
    from PIL import Image
    im = Image.fromarray(arr)
    if mode != im.mode:
        im = im.convert(mode)
    bio = io.BytesIO()
    im.save(bio, "PNG", **kw)
    return bio.getvalue()


def _replace_crc(blob, ty, delta=1, nth=0):
    """the file with the CRC of the nth chunk of type ty changed"""
    i, k = 8, 0
    b = bytearray(blob)
    while i < len(b):
        n = int.from_bytes(b[i:i + 4], "big")
        if bytes(b[i + 4:i + 8]) == ty:
            if k == nth:
                j = i + 8 + n
                b[j + 3] = (b[j + 3] + delta) & 255
                return bytes(b)
            k += 1
        i += 12 + n
    raise ValueError(ty)


def corpus(seed=0):
    """list of (name, bytes)"""
    rng = np.random.default_rng(seed)
    out = []
    # every colour type and bit depth, with and without Adam7, all five filters in turn
    for ct, depths in E.DEPTHS.items():
        for d in depths:
            for il in (False, True):
                h, w = int(rng.integers(1, 40)), int(rng.integers(1, 40))
                s = E.random_samples(rng, h, w, ct, d, smooth=bool(rng.integers(0, 2)))
                pal = None
                if ct == 3:
                    npal = int(rng.integers(1, (1 << d) + 1))
                    pal = rng.integers(0, 256, (npal, 3))
                out.append(("enc_c%d_d%d_i%d" % (ct, d, il), E.encode(s, ct, d, il, palette=pal)))
    # Adam7 on images with empty passes
    for h, w in ((1, 1), (1, 5), (3, 1), (2, 7), (7, 2), (5, 5), (8, 3), (9, 9)):
        out.append(("adam7_%dx%d" % (h, w), E.encode(E.random_samples(rng, h, w, 2, 8), 2, 8, True)))
    # filters chosen at random per row, wide bytes per pixel
    for ct, d in ((6, 16), (2, 16), (4, 8), (0, 1)):
        s = E.random_samples(rng, 23, 31, ct, d)
        out.append(("randfilter_c%d_d%d" % (ct, d), E.encode(s, ct, d, filters="random", rng=rng)))
    # zlib levels, strategies, window sizes; IDAT split points
    base = E.random_samples(rng, 37, 61, 2, 8)
    for lv in range(10):
        out.append(("level%d" % lv, E.encode(base, 2, 8, level=lv)))
    for name, st in (("filtered", zlib.Z_FILTERED), ("huffman", zlib.Z_HUFFMAN_ONLY), ("rle", zlib.Z_RLE), ("fixed", zlib.Z_FIXED)):
        out.append(("strategy_" + name, E.encode(base, 2, 8, strategy=st)))
    for wb in range(9, 16):
        out.append(("wbits%d" % wb, E.encode(E.random_samples(rng, 60, 200, 2, 8), 2, 8, wbits=wb, level=9)))
    out.append(("idat_split", E.encode(base, 2, 8, cuts=(1, 2, 2, 17, 300, 300))))
    out.append(("idat_zero_len", E.encode(base, 2, 8, cuts=(0, 0, 50))))
    # ancillary chunks and orientation
    text = E.chunk(b"tEXt", b"Comment\0hello")
    gama = E.chunk(b"gAMA", struct.pack(">I", 45455))
    small = E.random_samples(rng, 5, 9, 2, 8)
    out.append(("text_gama", E.encode(small, 2, 8, before=(text, gama), after=(text,))))
    for o in range(1, 9):
        be = bool(o % 2)
        ex = E.chunk(b"eXIf", E.exif_tiff(o, be))
        out.append(("exif%d_%s" % (o, "before" if o < 5 else "after"), E.encode(small, 2, 8, before=(ex,) if o < 5 else (), after=(ex,) if o >= 5 else ())))
    out.append(("exif6_2x1", E.encode(E.random_samples(rng, 1, 2, 2, 8), 2, 8, before=(E.chunk(b"eXIf", E.exif_tiff(6)),))))
    out.append(("exif6_bad_crc", _replace_crc(E.encode(small, 2, 8, before=(E.chunk(b"eXIf", E.exif_tiff(6)),)), b"eXIf")))
    out.append(("text_bad_crc", _replace_crc(E.encode(small, 2, 8, before=(text,)), b"tEXt")))
    out.append(("iend_bad_crc", _replace_crc(E.encode(small, 2, 8), b"IEND")))
    # palette edge cases
    idx = rng.integers(0, 16, (6, 11, 1))
    out.append(("pal_short", E.encode(idx, 3, 4, palette=rng.integers(0, 256, (5, 3)))))
    out.append(("pal_trns", E.encode(idx, 3, 4, palette=rng.integers(0, 256, (16, 3)), trns=bytes(range(16)))))
    out.append(("grey16_high", E.encode(np.full((2, 3, 1), 0x12FF), 0, 16)))
    # APNG
    z = E.compress(E.raw_data(small, 2, 8))
    out.append(("apng_idat_frame", E.encode(small, 2, 8, before=(E.actl(2), E.fctl(0, 9, 5)), after=(E.fctl(1, 9, 5), E.fdat(2, z)))))
    # deflate streams zlib does not emit
    raw = E.raw_data(E.random_samples(rng, 4, 6, 0, 8), 0, 8, filters=0)
    toks = list(raw) + ["end"]
    out.append(("defl_no_dist", _g4x6(raw, E.deflate_dynamic([toks]))))
    one = [raw[0]] + [("m", len(raw) - 1, 1)] + ["end"]
    rawone = E.tokens_to_bytes(one)
    out.append(("defl_one_dist", _g(rawone, 1, len(rawone) - 1, E.deflate_dynamic([one]))))
    # 4 rows of 16,383 grey bytes: a row with its filter byte is 16,384 bytes, so distance 32,768 is two rows up
    far = bytearray(rng.integers(0, 256, 32768, dtype=np.uint8))
    far[0] = far[16384] = 0
    long_toks = list(far) + [("m", 258, 32768)] * 126 + [("m", 257, 32768), ("m", 3, 32768), "end"]
    rawfar = E.tokens_to_bytes(long_toks)
    out.append(("defl_258_at_32768", _g(rawfar, 4, 16383, E.deflate_dynamic([long_toks]))))
    out.append(("defl_stored_0_65535", _g(bytes(65536), 4, 16383, E.deflate_stored([b"", b"", bytes(65535), b"\0"]))))
    # files of cv2 and PIL
    img = E.random_samples(rng, 33, 47, 2, 8).astype(np.uint8)
    for c in (0, 1, 5, 9):
        out.append(("cv2_comp%d" % c, cv2_encode(img, c)))
    for s in range(5):
        out.append(("cv2_strategy%d" % s, cv2_encode(img, 6, strategy=s)))
    for f in (8, 16, 32, 64, 128, 248):
        out.append(("cv2_filter%d" % f, cv2_encode(img, 6, filt=f)))
    out.append(("cv2_bilevel", cv2_encode((img[:, :, 0] > 127).astype(np.uint8) * 255, bilevel=True)))
    out.append(("cv2_gray16", cv2_encode((img[:, :, 0].astype(np.uint16) * 257 + 3))))
    out.append(("cv2_bgra", cv2_encode(np.concatenate([img, img[:, :, :1]], -1))))
    rgb = img[:, :, ::-1].copy()
    out.append(("pil_P", pil_encode(rgb, "P")))
    out.append(("pil_P_trns", pil_encode(rgb, "P", transparency=3)))
    out.append(("pil_1", pil_encode(rgb, "1")))
    out.append(("pil_L", pil_encode(rgb, "L")))
    out.append(("pil_LA", pil_encode(rgb, "LA")))
    out.append(("pil_I16", pil_encode((img[:, :, 0].astype(np.uint16) * 211), "I;16")))
    out.append(("pil_RGBA_opt", pil_encode(rgb, "RGBA", optimize=True)))
    return out + [(n, b) for n, b, _ in after_rows(seed)] + broken(seed)


def _two_blocks(toks, tail):
    """a non-final dynamic block of toks, then whatever tail(writer) writes"""
    w = E.BitWriter()
    ll, dl = E.lengths_for(toks)
    w.put(0, 1)
    w.put(2, 2)
    E.dynamic_header(w, ll, dl)
    E.write_tokens(w, toks, ll, dl)
    tail(w)
    return w.data()


def after_rows(seed=0):
    """(name, bytes, expected status or None for an image) of the streams that go on after the rows' data, as libpng
    reads them (each settled against cv2): data past the rows, the stream's end cut off after it, bytes after the stream,
    deflate errors before and after a byte past the rows is asked for; and distances past the window the zlib header
    declares (zlib refuses a source outside the current row call and its window)"""
    rng = np.random.default_rng(seed + 11)
    s = E.random_samples(rng, 20, 30, 2, 8)
    raw = E.raw_data(s, 2, 8)
    out = []
    for k in (3, 5000):
        z = E.compress(raw + bytes(rng.integers(0, 256, k, dtype=np.uint8)))
        out += [("extra%d" % k, E.encode(s, 2, 8, zdata=z), None),
                ("extra%d_bad_adler" % k, E.encode(s, 2, 8, zdata=z[:-1] + bytes([z[-1] ^ 1])), None),
                ("extra%d_no_adler" % k, E.encode(s, 2, 8, zdata=z[:-4]), 16),
                ("extra%d_cut" % k, E.encode(s, 2, 8, zdata=z[:-200] if len(z) > 400 else z[:-3]), 16)]
    z = E.compress(raw)
    out += [("trailing_bytes", E.encode(s, 2, 8, zdata=z + b"trailing garbage"), None),
            ("adler_cut", E.encode(s, 2, 8, zdata=z[:-2]), 16)]
    bad_type = lambda w: (w.put(1, 1), w.put(3, 2), w.put(0, 16))  # noqa: E731
    out += [("rows_then_bad_block", E.encode(s, 2, 8, zdata=E.zlib_wrap(_two_blocks(list(raw) + ["end"], bad_type), raw)), 16),
            ("extra_then_bad_block", E.encode(s, 2, 8, zdata=E.zlib_wrap(_two_blocks(list(raw) + [7, 7, "end"], bad_type), raw)), None),
            ("extra_match_too_far", E.encode(s, 2, 8, zdata=E.zlib_wrap(E.deflate_dynamic([list(raw) + [("m", 3, len(raw) + 50), "end"]]),
                                                                        raw)), None)]
    # 2 x 999 grey: the second row copies the first at distance 1,000 (windows of 256 and 512 bytes refuse it)
    row = bytes([0]) + bytes(rng.integers(0, 256, 999, dtype=np.uint8))
    toks = list(row) + [("m", 258, 1000)] * 3 + [("m", 226, 1000), "end"]
    for ci in (0, 1, 2, 7):
        out.append(("window%d_d1000" % ci, E.encode(np.zeros((2, 999, 1)), 0, 8, zdata=E.zlib_wrap(E.deflate_dynamic([toks]),
                                                                                                   E.tokens_to_bytes(toks), cinfo=ci)),
                    16 if ci < 2 else None))
    # rows of 100 bytes, a 256-byte window: a distance of 290 reaches back within its row call, but not into the next row
    rows = [bytearray([0]) + bytearray(rng.integers(0, 256, 99, dtype=np.uint8)) for _ in range(3)]
    rows[1][10] = 0
    head = list(bytes(rows[0] + rows[1] + rows[2])) + list(bytes(rows[0][:80]))
    for n, name, st in ((20, "window0_d290_in_row", None), (40, "window0_d290_next_row", 16)):
        toks = head + [("m", n, 290)] + ([0] + [int(v) for v in rng.integers(0, 256, 99)] if n == 20 else
                                         [int(v) for v in rng.integers(0, 256, 80)]) + ["end"]
        out.append((name, E.encode(np.zeros((5, 99, 1)), 0, 8, zdata=E.zlib_wrap(E.deflate_dynamic([toks]), E.tokens_to_bytes(toks),
                                                                                 cinfo=0)), st))
    return out


def _g(raw, h, w, deflate):
    """a grey 8-bit file of h x w (raw must be its filtered rows) over a hand-made deflate stream"""
    return E.encode(np.zeros((h, w, 1)), 0, 8, zdata=E.zlib_wrap(deflate, raw))


def _g4x6(raw, deflate):
    return _g(raw, 4, 6, deflate)


def broken(seed=0):
    rng = np.random.default_rng(seed + 7)
    s = E.random_samples(rng, 20, 30, 2, 8)
    good = E.encode(s, 2, 8)
    raw = E.raw_data(s, 2, 8)
    z = E.compress(raw)
    out = [("not_png", b"\xff\xd8\xff\xe0" + bytes(40)),
           ("short_sig", good[:6]),
           ("bad_ihdr_crc", _replace_crc(good, b"IHDR")),
           ("bad_idat_crc", _replace_crc(E.encode(s, 2, 8, cuts=(100,)), b"IDAT", nth=1)),
           ("bad_plte_crc", _replace_crc(E.encode(rng.integers(0, 4, (4, 4, 1)), 3, 2, palette=[[1, 2, 3]] * 4), b"PLTE")),
           ("no_iend", good[:-12]),
           ("truncated_chunk", good[:len(good) // 2]),
           ("no_plte", E.encode(rng.integers(0, 4, (4, 4, 1)), 3, 2)),
           ("bad_depth", good[:24] + bytes([3]) + good[25:29] + struct.pack(">I", zlib.crc32(good[12:16] + good[16:24] + bytes([3]) + good[25:29])) + good[33:]),
           ("idat_interrupted", _interrupt(good)),
           ("bad_adler", E.encode(s, 2, 8, zdata=z[:-4] + bytes([z[-4] ^ 1]) + z[-3:])),
           ("zlib_truncated", E.encode(s, 2, 8, zdata=z[:len(z) // 2])),
           ("zlib_no_adler", E.encode(s, 2, 8, zdata=z[:-4])),
           ("zlib_bad_header", E.encode(s, 2, 8, zdata=bytes([0x78, 0x9D]) + z[2:])),
           ("zlib_cinfo8", E.encode(s, 2, 8, zdata=_zhdr(0x88, 0) + z[2:])),
           ("zlib_fdict", E.encode(s, 2, 8, zdata=_zhdr(0x78, 0x20) + z[2:])),
           ("bad_block_type", _g(raw[:31], 1, 30, _blocktype3())),
           ("oversubscribed", _g(raw[:31], 1, 30, _oversub())),
           ("dist_too_far", _g(bytes(31), 1, 30, E.deflate_dynamic([[0, ("m", 10, 5), "end"]]))),
           ("short_data", E.encode(s, 2, 8, zdata=E.compress(raw[:-5]))),
           ("bad_filter", E.encode(s, 2, 8, zdata=E.compress(bytes([7]) + raw[1:]))),
           ("apng_idat_not_frame", E.encode(s, 2, 8, before=(E.actl(1),), after=(E.fctl(0, 30, 20), E.fdat(1, z))))]
    return out


def _zhdr(cmf, flags):
    """a zlib header with a valid FCHECK"""
    return bytes([cmf, flags + (31 - ((cmf << 8) + flags) % 31) % 31])


def _interrupt(good):
    """the IDAT data split in two chunks with a tEXt chunk between"""
    s = E.random_samples(np.random.default_rng(5), 20, 30, 2, 8)
    z = E.compress(E.raw_data(s, 2, 8))
    a, b = z[:len(z) // 2], z[len(z) // 2:]
    f = E.SIG + E.chunk(b"IHDR", struct.pack(">IIBBBBB", 30, 20, 8, 2, 0, 0, 0))
    return f + E.chunk(b"IDAT", a) + E.chunk(b"tEXt", b"a\0b") + E.chunk(b"IDAT", b) + E.chunk(b"IEND", b"")


def _blocktype3():
    w = E.BitWriter()
    w.put(1, 1)
    w.put(3, 2)
    w.put(0, 16)
    return w.data()


def _oversub():
    w = E.BitWriter()
    w.put(1, 1)
    w.put(2, 2)
    E.dynamic_header(w, [1] * 257, [1], cl_override=[1] * 19)
    return w.data()


EXPECTED_STATUS = dict(not_png=1, short_sig=1, bad_ihdr_crc=1, bad_idat_crc=1, bad_plte_crc=1, no_iend=1, truncated_chunk=1,
                       no_plte=1, bad_depth=1, idat_interrupted=1, bad_adler=16, zlib_truncated=16, zlib_no_adler=16,
                       zlib_bad_header=16, zlib_cinfo8=16, zlib_fdict=16, bad_block_type=16, oversubscribed=16,
                       dist_too_far=16, short_data=16, bad_filter=16, apng_idat_not_frame=2,
                       **{n: st for n, _, st in after_rows() if st is not None})


def random_case(rng):
    """one random PNG: colour type, depth, size, interlace, filters, zlib level / strategy, IDAT splits; one in six with
    data past the rows in its zlib stream"""
    ct = int(rng.choice(list(E.DEPTHS)))
    d = int(rng.choice(E.DEPTHS[ct]))
    h, w = int(rng.integers(1, 70)), int(rng.integers(1, 90))
    s = E.random_samples(rng, h, w, ct, d, smooth=bool(rng.integers(0, 2)))
    pal = rng.integers(0, 256, (int(rng.integers(1, (1 << d) + 1)), 3)) if ct == 3 else None
    st = int(rng.choice([zlib.Z_DEFAULT_STRATEGY, zlib.Z_FILTERED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE, zlib.Z_FIXED]))
    cuts = rng.integers(0, 400, int(rng.integers(0, 4)))
    il, level, wbits = bool(rng.integers(0, 2)), int(rng.integers(0, 10)), int(rng.integers(9, 16))
    if rng.random() < 1 / 6:
        raw = E.raw_data(s, ct, d, il, "random", rng) + bytes(rng.integers(0, 256, int(rng.integers(1, 3000)), dtype=np.uint8))
        return E.encode(s, ct, d, il, cuts=cuts, palette=pal, zdata=E.compress(raw, level, st, wbits))
    return E.encode(s, ct, d, il, filters="random", rng=rng, level=level, strategy=st, wbits=wbits, cuts=cuts, palette=pal)
