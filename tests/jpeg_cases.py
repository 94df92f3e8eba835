"""Seeded JPEG inputs of the decoder tests and the host harness (tests/host_harness/jpeg_core_host.cpp, the product's
jpeg_core.cuh compiled with g++).

corpus() encodes with cv2 (4:4:4, 4:2:2, 4:2:0, 4:4:0, 4:1:1 and grey, qualities 1 to 100, optimised tables, restart
intervals 1 / 2 / 3 / 64, sides 1 to a few hundred) and with PIL (Adobe transform 0 via keep_rgb, EXIF orientations 1 to 8,
grey, CMYK, progressive), and adds edited files: a big-endian EXIF, 16-bit quantisation tables, fill bytes and a COM
segment, a lossless SOF, RSTn out of order, truncated headers and scans, and bytes that are not a JPEG; crafted() adds the
files of the numpy baseline encoder (tests/jpeg_encoder.py)."""
import ctypes
import io
import os
import shutil
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "megreader_b200", "csrc")

SAMPLING = {"444": 0x111111, "422": 0x211111, "420": 0x221111, "440": 0x121111, "411": 0x411111}


def build_sanitized(tmp):
    """the harness as an executable under AddressSanitizer and UBSan (decodes the files named on its command line), or
    None where g++ cannot build one"""
    gxx = shutil.which("g++")
    if gxx is None:
        return None
    exe = os.path.join(str(tmp), "jpeg_core_host_asan")
    cmd = [gxx, "-O1", "-g", "-std=c++17", "-ffp-contract=off", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
           "-fno-omit-frame-pointer", "-DJPEG_HARNESS_MAIN", "-I" + CSRC, os.path.join(HERE, "host_harness", "jpeg_core_host.cpp"),
           "-o", exe]
    if subprocess.run(cmd, capture_output=True).returncode != 0:
        return None
    return exe


def build_harness(tmp):
    gxx = shutil.which("g++")
    if gxx is None:
        return None
    so = os.path.join(str(tmp), "libjpeg_core_host.so")
    subprocess.check_call([gxx, "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-I" + CSRC,
                           os.path.join(HERE, "host_harness", "jpeg_core_host.cpp"), "-o", so])
    L = ctypes.CDLL(so)
    P, I64 = ctypes.c_void_p, ctypes.c_int64
    L.host_header.argtypes = [P, I64, P]
    L.host_decode.argtypes = [P, I64, ctypes.c_int, I64, P, P, P]
    L.host_coefs.argtypes = [P, I64, ctypes.c_int, I64, P, P, P]
    L.host_coefs.restype = I64
    return L


def host_decode(L, blob, run_bits=0):
    """(status, HWC uint8 array or None, runs the walker decoded) of the product's routines on one byte string"""
    b = np.frombuffer(bytes(blob), np.uint8)
    info = np.zeros(8, np.int32)
    L.host_header(b.ctypes.data, b.size, info.ctypes.data)
    cap = max(3 * int(info[1]) * int(info[2]), 1)
    out = np.zeros(cap, np.uint8)
    hw = np.zeros(2, np.int32)
    fixed = np.zeros(1, np.int32)
    st = L.host_decode(b.ctypes.data, b.size, run_bits, cap, out.ctypes.data, hw.ctypes.data, fixed.ctypes.data)
    if st:
        return st, None, int(fixed[0])
    return 0, out[:3 * hw[0] * hw[1]].reshape(hw[0], hw[1], 3), int(fixed[0])


def image(rng, h, w, kind="smooth"):
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == "flat":
        return np.full((h, w, 3), rng.integers(0, 256, 3), np.uint8)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    f = rng.uniform(3, 20, 3)
    base = np.stack([127 + 90 * np.sin(x / f[c] + c) * np.cos(y / (f[c] + 3) - c) for c in range(3)], -1)
    base += rng.normal(0, 10, (h, w, 3))
    return np.clip(base, 0, 255).astype(np.uint8)


def cv2_encode(img, quality=90, sampling="420", optimize=False, rst=0):
    import cv2
    p = [cv2.IMWRITE_JPEG_QUALITY, int(quality)]
    if img.ndim == 3:
        p += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, SAMPLING[sampling]]
    if optimize:
        p += [cv2.IMWRITE_JPEG_OPTIMIZE, 1]
    if rst:
        p += [cv2.IMWRITE_JPEG_RST_INTERVAL, int(rst)]
    ok, b = cv2.imencode(".jpg", img, p)
    assert ok
    return b.tobytes()


def pil_encode(img, **kw):
    from PIL import Image
    bio = io.BytesIO()
    mode = kw.pop("mode", None)
    im = Image.fromarray(img[:, :, ::-1] if img.ndim == 3 else img)
    if mode is not None and mode != im.mode:
        im = im.convert(mode)
    im.save(bio, "JPEG", **kw)
    return bio.getvalue()


def exif_bytes(orientation, big_endian=False):
    if big_endian:
        tiff = b"MM\x00\x2a" + (8).to_bytes(4, "big") + (1).to_bytes(2, "big")
        tiff += (0x0112).to_bytes(2, "big") + (3).to_bytes(2, "big") + (1).to_bytes(4, "big") + orientation.to_bytes(2, "big") + b"\0\0"
    else:
        tiff = b"II\x2a\x00" + (8).to_bytes(4, "little") + (1).to_bytes(2, "little")
        tiff += (0x0112).to_bytes(2, "little") + (3).to_bytes(2, "little") + (1).to_bytes(4, "little")
        tiff += orientation.to_bytes(2, "little") + b"\0\0"
    return b"Exif\x00\x00" + tiff + (0).to_bytes(4, "little")


def insert_after_soi(blob, seg_marker, payload):
    return blob[:2] + bytes([0xFF, seg_marker]) + (len(payload) + 2).to_bytes(2, "big") + payload + blob[2:]


def segments(blob):
    """(marker, start, end) of every marker segment before SOS, and the SOS's"""
    out, i = [], 2
    while i < len(blob):
        m = blob[i + 1]
        n = int.from_bytes(blob[i + 2:i + 4], "big")
        out.append((m, i, i + 2 + n))
        if m == 0xDA:
            break
        i += 2 + n
    return out


def dqt16(blob):
    """the same image with its 8-bit quantisation tables rewritten as 16-bit ones (same values)"""
    res = bytearray()
    last = 0
    for m, s, e in segments(blob):
        if m != 0xDB:
            continue
        res += blob[last:s]
        body, j, new = blob[s + 4:e], 0, bytearray()
        while j < len(body):
            pq, tq = body[j] >> 4, body[j] & 15
            vals = body[j + 1:j + 1 + (128 if pq else 64)]
            vals = np.frombuffer(vals, ">u2") if pq else np.frombuffer(vals, np.uint8)
            new += bytes([0x10 | tq]) + vals.astype(">u2").tobytes()
            j += 1 + (128 if pq else 64)
        res += b"\xff\xdb" + (len(new) + 2).to_bytes(2, "big") + new
        last = e
    return bytes(res + blob[last:])


def corpus(seed=0):
    """list of (name, bytes): the decoder's seeded test corpus"""
    rng = np.random.default_rng(seed)
    out = []
    sides = [1, 2, 3, 7, 8, 9, 15, 16, 17]
    for samp in SAMPLING:
        for h in sides:
            w = int(rng.choice(sides))
            out.append(("cv2_%s_%dx%d" % (samp, h, w), cv2_encode(image(rng, h, w), int(rng.integers(1, 101)), samp)))
        for rst in (1, 3, 64):
            h, w = int(rng.integers(20, 200)), int(rng.integers(20, 300))
            out.append(("cv2_%s_rst%d" % (samp, rst), cv2_encode(image(rng, h, w), int(rng.integers(50, 101)), samp, rst=rst)))
        h, w = int(rng.integers(100, 400)), int(rng.integers(100, 400))
        out.append(("cv2_%s_opt" % samp, cv2_encode(image(rng, h, w), 85, samp, optimize=True)))
    for q in (1, 5, 25, 50, 75, 95, 100):
        out.append(("cv2_q%d" % q, cv2_encode(image(rng, 61, 83), q, "420")))
    out.append(("cv2_noise_q100", cv2_encode(image(rng, 40, 70, "noise"), 100, "444")))
    out.append(("cv2_flat", cv2_encode(image(rng, 120, 200, "flat"), 90, "420")))
    for h in (1, 7, 16, 33):
        out.append(("cv2_gray_%d" % h, cv2_encode(image(rng, h, 45)[:, :, 0], 80)))
    out.append(("cv2_gray_rst2", cv2_encode(image(rng, 50, 66)[:, :, 0], 80, rst=2)))
    base = image(rng, 37, 53)
    for o in range(1, 9):
        out.append(("pil_exif%d" % o, insert_after_soi(pil_encode(base, quality=90), 0xE1, exif_bytes(o))))
    out.append(("exif6_big_endian", insert_after_soi(pil_encode(base, quality=90), 0xE1, exif_bytes(6, True))))
    out.append(("pil_keep_rgb", pil_encode(base, quality=90, keep_rgb=True)))
    out.append(("pil_440", pil_encode(base, quality=90, subsampling="4:4:0") if _pil_has_440() else cv2_encode(base, 90, "440")))
    out.append(("pil_gray", pil_encode(base[:, :, 0], quality=70)))
    out.append(("dqt16", dqt16(cv2_encode(image(rng, 30, 41), 60, "422"))))
    out.append(("fill_bytes", _fill_bytes(cv2_encode(image(rng, 24, 24), 80, "444"))))
    # unsupported or broken
    out.append(("pil_cmyk", pil_encode(base, quality=90, mode="CMYK")))
    out.append(("pil_progressive", pil_encode(base, quality=90, progressive=True)))
    good = cv2_encode(image(rng, 64, 96), 90, "420")
    out.append(("truncated_scan", good[:len(good) * 2 // 3]))
    out.append(("truncated_header", good[:100]))
    out.append(("not_jpeg", b"\x89PNG\r\n\x1a\n" + bytes(rng.integers(0, 256, 50, dtype=np.uint8))))
    out.append(("lossless_sof3", good.replace(b"\xff\xc0", b"\xff\xc3", 1)))
    out.append(("bad_rst_order", _swap_rst(cv2_encode(image(rng, 48, 64), 90, "420", rst=1))))
    return out + crafted(seed)


def _blocks(rng, ncomp, h, w, scale, dc_only=False):
    b = np.round(rng.normal(0, scale, (ncomp, (h + 7) // 8, (w + 7) // 8, 8, 8))).astype(int)
    b *= rng.random(b.shape) > 0.7
    if dc_only:
        b[:] = 0
        b[..., 0, 0] = rng.integers(-2047, 2048, b.shape[:3])
    return np.clip(b, -32767, 32767)


def crafted(seed=0):
    """files of tests/jpeg_encoder.py: IDCT values past 16 bits (16-bit quantisation tables up to 65535, coefficients up to
    about +-10,000, DC-only blocks whose dequantised DC wraps), Huffman tables with 16-bit codes, and the headers the
    decoder refuses (names in REFUSED, with their status)"""
    from tests import jpeg_encoder as E
    rng = np.random.default_rng(seed + 100)
    q = lambda n, lo, hi: rng.integers(lo, hi, (n, 64))  # noqa: E731
    out = []
    for i in range(3):
        out.append(("enc_q16x8_%d" % i, E.encode(_blocks(rng, 3, 40, 56, 3), q(3, 8, 800), 40, 56, dqt16=True)))
        out.append(("enc_q16big_%d" % i, E.encode(_blocks(rng, 3, 23, 41, 4), q(3, 1000, 65536), 23, 41, dqt16=True)))
        out.append(("enc_hugecoef_%d" % i, E.encode(_blocks(rng, 1, 24, 24, 3000), q(1, 1, 40), 24, 24, dqt16=True)))
        out.append(("enc_dconly_%d" % i, E.encode(_blocks(rng, 3, 24, 40, 1, dc_only=True), q(3, 1, 256), 24, 40)))
        out.append(("enc_long_codes_%d" % i, E.encode(_blocks(rng, 3, 33, 47, 5), q(3, 1, 60), 33, 47, long_codes=True)))
    out.append(("enc_sof1_grey", E.encode(_blocks(rng, 1, 17, 9, 30), q(1, 1, 256), 17, 9, marker=0xC1)))
    three = ((1, 1, 1, 0), (2, 1, 1, 0), (3, 1, 1, 0))
    out += [("hdr_progressive", E.header_only(0xC2)), ("hdr_lossless", E.header_only(0xC3)),
            ("hdr_hierarchical", E.header_only(0xC5)), ("hdr_arithmetic", E.header_only(0xC9)),
            ("hdr_12bit", E.header_only(0xC1, precision=12)), ("hdr_dnl", E.header_only(h=0)),
            ("hdr_multiscan", E.header_only(comps=three, scan_ids=[1])),
            ("hdr_2comp", E.header_only(comps=three[:2])), ("hdr_4comp", E.header_only(comps=three + ((4, 1, 1, 0),))),
            ("hdr_fractional", E.header_only(comps=((1, 3, 1, 0), (2, 2, 1, 0), (3, 1, 1, 0))))]
    return out


REFUSED = dict(hdr_progressive=2, hdr_lossless=2, hdr_hierarchical=2, hdr_arithmetic=2, hdr_12bit=2, hdr_dnl=2, hdr_multiscan=2,
               hdr_2comp=4, hdr_4comp=4, hdr_fractional=4)


def _pil_has_440():
    try:
        from PIL import JpegImagePlugin  # noqa: F401
        pil_encode(np.zeros((8, 8, 3), np.uint8), subsampling="4:4:0")
        return True
    except Exception:
        return False


def _fill_bytes(blob):
    """0xFF fill bytes before every marker after SOI, and a COM segment"""
    res = bytearray(blob[:2]) + b"\xff\xfe\x00\x05abc"
    last = 2
    for m, s, e in segments(blob):
        res += blob[last:s] + b"\xff\xff"
        last = s
    return bytes(res + blob[last:])


def _swap_rst(blob):
    i = blob.index(b"\xff\xd0", 200)
    j = blob.index(b"\xff\xd1", i)
    b = bytearray(blob)
    b[i + 1], b[j + 1] = 0xD1, 0xD0
    return bytes(b)


def random_case(rng):
    """one random (bytes, params) of random size, sampling, quality and restart interval"""
    h, w = int(rng.integers(1, 120)), int(rng.integers(1, 160))
    samp = str(rng.choice(list(SAMPLING) + ["gray"]))
    img = image(rng, h, w, str(rng.choice(["smooth", "noise", "flat"], p=[0.7, 0.2, 0.1])))
    q = int(rng.integers(1, 101))
    rst = int(rng.choice([0, 0, 1, 2, 5, 17]))
    opt = bool(rng.integers(0, 2))
    if samp == "gray":
        return cv2_encode(img[:, :, 0], q, optimize=opt, rst=rst)
    return cv2_encode(img, q, samp, optimize=opt, rst=rst)
