"""CPU: the PRODUCT's JPEG routines (megreader_b200/csrc/jpeg_core.cuh -- the code the CUDA kernels of csrc/jpeg.cu run)
compiled for the host by tests/host_harness/jpeg_core_host.cpp, checked against cv2.imdecode(buf, cv2.IMREAD_COLOR) live:
  * the seeded corpus of tests/jpeg_cases.py, bit for bit, and the status of every unsupported or broken file; it includes
    the numpy baseline encoder's files (tests/jpeg_encoder.py): IDCT values past 16 bits, where libjpeg-turbo's SIMD IDCT
    (which cv2 runs) wraps and saturates, 16-bit quantisation tables with large values, 16-bit Huffman codes, and the
    headers of the processes and component layouts the decoder refuses;
  * 1,000 more seeded images of random size, sampling, quality, table optimisation and restart interval;
  * the synchronising run decode of jpeg.cu as a host loop at small run sizes gives the sequential decode's coefficients;
  * the corrupt inputs once more under AddressSanitizer and UBSan, where the toolchain has them."""
import os
import subprocess

import numpy as np
import pytest

from tests import jpeg_cases as C

cv2 = pytest.importorskip("cv2")


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    L = C.build_harness(tmp_path_factory.mktemp("harness"))
    if L is None:
        pytest.skip("g++ not available")
    return L


@pytest.fixture(scope="module")
def corpus():
    return C.corpus()


def _cv2(blob):
    return cv2.imdecode(np.frombuffer(blob, np.uint8), cv2.IMREAD_COLOR)


EXPECTED_STATUS = dict(pil_cmyk=4, pil_progressive=2, truncated_header=1, not_jpeg=1, lossless_sof3=2, bad_rst_order=16,
                       truncated_scan=16, **C.REFUSED)


@pytest.mark.parametrize("run_bits", [0, 64])
def test_corpus_bit_exact(lib, corpus, run_bits):
    exact = 0
    for name, blob in corpus:
        st, out, _ = C.host_decode(lib, blob, run_bits)
        if name in EXPECTED_STATUS:
            assert st == EXPECTED_STATUS[name], (name, st)
            continue
        ref = _cv2(blob)
        assert st == 0 and ref is not None, (name, st)
        assert out.shape == ref.shape and np.array_equal(out, ref), name
        exact += 1
    assert exact >= 95


def test_random_images_bit_exact(lib):
    rng = np.random.default_rng(2024)
    for i in range(1000):
        blob = C.random_case(rng)
        st, out, _ = C.host_decode(lib, blob, int(rng.choice([0, 40, 512])))
        ref = _cv2(blob)
        assert st == 0 and out.shape == ref.shape and np.array_equal(out, ref), i


def test_headers(lib, corpus):
    d = dict(corpus)
    info = np.zeros(8, np.int32)
    for o in range(1, 9):
        b = np.frombuffer(d["pil_exif%d" % o], np.uint8)
        lib.host_header(b.ctypes.data, b.size, info.ctypes.data)
        assert info[4] == o and tuple(info[1:3]) == ((53, 37) if o >= 5 else (37, 53))
    for name, cs in (("pil_keep_rgb", 2), ("cv2_420_opt", 1), ("pil_gray", 0)):
        b = np.frombuffer(d[name], np.uint8)
        lib.host_header(b.ctypes.data, b.size, info.ctypes.data)
        assert info[3] == cs, name


@pytest.mark.parametrize("run_bits", [8, 17, 32, 100])
def test_sync_decode_equals_sequential(lib, run_bits):
    rng = np.random.default_rng(run_bits)
    cases = [C.cv2_encode(C.image(rng, 64, 80, "flat"), 90, "420"),             # flat: many blocks per run
             C.cv2_encode(C.image(rng, 40, 56, "noise"), 100, "444"),           # noise at q100: long codes
             C.cv2_encode(C.image(rng, 50, 70), 75, "422", rst=1),               # restart interval 1
             C.cv2_encode(C.image(rng, 1, 1), 50, "420")]                        # a scan shorter than one run
    cases += [C.random_case(rng) for _ in range(40)]
    for blob in cases:
        b = np.frombuffer(blob, np.uint8)
        cap = 64 * 10 * 4096
        a, s = np.zeros(cap, np.int16), np.zeros(cap, np.int16)
        fixed = np.zeros(1, np.int32)
        nb = lib.host_coefs(b.ctypes.data, b.size, run_bits, cap, a.ctypes.data, s.ctypes.data, fixed.ctypes.data)
        assert nb > 0
        np.testing.assert_array_equal(a[:64 * nb], s[:64 * nb])


def test_corrupt_inputs_under_sanitizers(tmp_path, corpus):
    exe = C.build_sanitized(tmp_path)
    if exe is None:
        pytest.skip("g++ cannot build with -fsanitize=address,undefined here")
    rng = np.random.default_rng(9)
    blobs = [b for n, b in corpus if n in EXPECTED_STATUS]
    good = C.cv2_encode(C.image(rng, 48, 64), 85, "420", rst=3)
    for _ in range(60):
        b = bytearray(good)
        for _ in range(int(rng.integers(1, 6))):
            b[int(rng.integers(2, len(b)))] = int(rng.integers(0, 256))
        blobs.append(bytes(b[:int(rng.integers(4, len(b) + 1))]))
    files = []
    for i, blob in enumerate(blobs):
        f = tmp_path / ("case%03d.jpg" % i)
        f.write_bytes(blob)
        files.append(str(f))
    r = subprocess.run([exe] + files, capture_output=True, text=True, env=dict(os.environ, ASAN_OPTIONS="detect_leaks=0"))
    assert r.returncode == 0, r.stderr[-3000:]
