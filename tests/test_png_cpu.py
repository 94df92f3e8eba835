"""CPU: the PRODUCT's PNG routines (megreader_b200/csrc/png_core.cuh -- the code the CUDA kernels of csrc/png.cu run) compiled
for the host by tests/host_harness/png_core_host.cpp, checked against cv2.imdecode(buf, cv2.IMREAD_COLOR) live:
  * the seeded corpus of tests/png_cases.py bit for bit, and the status of every broken file;
  * 1,000 more seeded random files;
  * the kernels' match resolution (recorded matches, pointer jumping) against the serial inflate's copies;
  * the corrupt files once more under AddressSanitizer and UBSan, where g++ has them;
  * the argument checks of the four C entries, without a GPU."""
import os
import subprocess

import numpy as np
import pytest

from tests import png_cases as C

cv2 = pytest.importorskip("cv2")


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    L = C.build_harness(tmp_path_factory.mktemp("png_harness"))
    if L is None:
        pytest.skip("g++ not available")
    return L


@pytest.fixture(scope="module")
def corpus():
    return C.corpus()


def _cv2(blob):
    return cv2.imdecode(np.frombuffer(blob, np.uint8), cv2.IMREAD_COLOR)


@pytest.mark.parametrize("jump", [0, 1])
def test_corpus_bit_exact(lib, corpus, jump):
    exact = 0
    for name, blob in corpus:
        st, out, _ = C.host_decode(lib, blob, jump)
        ref = _cv2(blob)
        if name in C.EXPECTED_STATUS:
            assert st == C.EXPECTED_STATUS[name], (name, st)
            if C.EXPECTED_STATUS[name] != 2:        # the one listed deviation: cv2 decodes the first fdAT frame
                assert ref is None, name
            continue
        assert ref is not None, name
        assert st == 0, (name, st)
        assert out.shape == ref.shape and np.array_equal(out, ref), name
        exact += 1
    assert exact >= 100


def test_random_files_bit_exact(lib):
    rng = np.random.default_rng(2025)
    for i in range(1000):
        blob = C.random_case(rng)
        st, out, _ = C.host_decode(lib, blob, int(i % 2))
        ref = _cv2(blob)
        assert st == 0 and out.shape == ref.shape and np.array_equal(out, ref), i


def test_headers(lib, corpus):
    d = dict(corpus)
    info = C.header(lib, d["exif6_2x1"])
    assert info[6] == 6 and tuple(info[1:3]) == (2, 1)
    assert C.header(lib, d["exif6_bad_crc"])[6] == 1
    for o in range(1, 9):
        info = C.header(lib, d["exif%d_%s" % (o, "before" if o < 5 else "after")])
        assert info[6] == o and tuple(info[1:3]) == ((9, 5) if o >= 5 else (5, 9))


def test_sides_zero_or_past_16384(lib):
    """an IHDR with a zero side is malformed for libpng and here (1); a side past 16384 is flagged 8 (cv2 decodes it)"""
    import struct
    from tests import png_encoder as E
    s = np.zeros((3, 4, 3), np.uint32)
    for w, h in ((0, 3), (4, 0)):
        b = E.encode(s, 2, 8, ihdr=struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 0))
        assert _cv2(b) is None and C.host_decode(lib, b)[0] == 1
    wide = E.encode(np.zeros((1, 16385, 1), np.uint32), 0, 8)
    assert _cv2(wide).shape == (1, 16385, 3) and C.host_decode(lib, wide)[0] == 8


def test_pointer_jumping_equals_serial_inflate(lib, corpus):
    """matches resolved from their records by pointer jumping give the serial copies; long chains take log2 rounds"""
    d = dict(corpus)
    for name in ("defl_258_at_32768", "defl_one_dist", "strategy_rle", "level9", "cv2_comp9", "wbits9"):
        a, b = C.host_decode(lib, d[name], 0), C.host_decode(lib, d[name], 1)
        assert a[0] == b[0] == 0 and np.array_equal(a[1], b[1]), name
    _, _, rounds = C.host_decode(lib, d["defl_one_dist"], 1)
    assert 1 <= rounds <= 7


def test_corrupt_inputs_under_sanitizers(tmp_path, corpus):
    exe = C.build_sanitized(tmp_path)
    if exe is None:
        pytest.skip("g++ cannot build with -fsanitize=address,undefined here")
    rng = np.random.default_rng(9)
    blobs = [b for n, b in corpus if n in C.EXPECTED_STATUS]
    good = dict(corpus)["level6"]
    for _ in range(80):
        b = bytearray(good)
        for _ in range(int(rng.integers(1, 6))):
            b[int(rng.integers(8, len(b)))] = int(rng.integers(0, 256))
        blobs.append(bytes(b[:int(rng.integers(4, len(b) + 1))]))
    files = []
    for i, blob in enumerate(blobs):
        f = tmp_path / ("case%03d.png" % i)
        f.write_bytes(blob)
        files.append(str(f))
    r = subprocess.run([exe] + files, capture_output=True, text=True, env=dict(os.environ, ASAN_OPTIONS="detect_leaks=0"))
    assert r.returncode == 0, r.stderr[-3000:]


def test_c_entries_argument_checks():
    """the four entries refuse bad sizes and short workspaces before any CUDA call"""
    from megreader_b200 import _lib
    L = _lib.lib()
    for ws, dec in (("mr_png_workspace_bytes", "mr_png_decode"), ("mr_image_workspace_bytes", "mr_image_decode")):
        assert getattr(L, ws)(0, 10, 10) == 0 and getattr(L, ws)(1, -1, 10) == 0 and getattr(L, ws)(70000, 10, 10) == 0
        need = getattr(L, ws)(2, 1000, 5000)
        assert need > 0
        p = 0x10000
        f = getattr(L, dec)
        assert f(p, 1000, p, 2, 16384, 16384, 5000, p, need - 1, p, p, p, p, None) == 4      # workspace too small
        assert f(p, 1000, p, 2, 0, 16384, 5000, p, need, p, p, p, p, None) == 4              # max_h outside 1..16384
        assert f(p, 1000, p, 0, 16384, 16384, 5000, p, need, p, p, p, p, None) == 4          # N = 0
        assert f(None, 1000, p, 2, 16384, 16384, 5000, p, need, p, p, p, p, None) == 1       # null data
