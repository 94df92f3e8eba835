"""TEST INFRASTRUCTURE ONLY (never imported by the product): CPU restatement of the recognition input step
(SURVEY.md section 8 row N3) as the reference's data pipeline runs it for `experiments/recognition/crnn.yaml`:

    image = cv2.imdecode(...).astype('float32')                 data/lmdb_dataset.py:87         (HWC, 3 channels)
    image = cv2.resize(image, (width, height))                  data/processes/resize_image.py:29-57 (modes resize / pad)
    image -= RGB_MEAN ; image /= 255. ; HWC -> CHW float32      data/processes/normalize_image.py:10-17
    label = charset.string_to_label(gt)[:max_size]; length      data/processes/make_recognition_label.py:13-32

cv2.resize is third-party (OpenCV 4.13 in this image, INTER_LINEAR on CV_32F): its published algorithm is restated in
`resize_bilinear_f32` — half-pixel centres, coefficients computed from scale = 1/(dst/src) in double and stored as float,
left/right neighbours clamped by forcing the fraction to 0, rows clamped by index.  Pinned by tests/test_oracle_input.py
against cv2 itself (<= 1e-4 on the 0..255 scale: OpenCV's SIMD path fuses some multiply-adds) and against the UNMODIFIED
reference processes (goldens tests/golden/input_ref.npz)."""
import numpy as np

RGB_MEAN = np.array([122.67891434, 116.66876762, 104.00698793])          # normalize_image.py:8


def _coeffs(dst, src):
    scale = 1.0 / (float(dst) / float(src))                                # cv::resize: scale = 1 / inv_scale (double)
    d = np.arange(dst, dtype=np.float64)
    f = ((d + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    return s, f


def resize_bilinear_f32(img, dst_h, dst_w):
    """img [H, W, C] float32 -> [dst_h, dst_w, C] float32 (cv2.resize(img, (dst_w, dst_h)), INTER_LINEAR)."""
    img = np.asarray(img, dtype=np.float32)
    H, W, _ = img.shape
    sx, fx = _coeffs(dst_w, W)
    lo = sx < 0
    fx[lo], sx[lo] = 0.0, 0
    hi = sx >= W - 1
    fx[hi], sx[hi] = 0.0, W - 1
    x1 = np.minimum(sx + 1, W - 1)
    a0, a1 = (np.float32(1.0) - fx)[None, :, None], fx[None, :, None]
    rows = img[:, sx, :] * a0 + img[:, x1, :] * a1                           # horizontal pass, float
    sy, fy = _coeffs(dst_h, H)
    y0, y1 = np.clip(sy, 0, H - 1), np.clip(sy + 1, 0, H - 1)               # vertical pass: index clamp only
    b0, b1 = (np.float32(1.0) - fy)[:, None, None], fy[:, None, None]
    return (rows[y0] * b0 + rows[y1] * b1).astype(np.float32)


def resized_width(mode, image_size, src_h, src_w):
    """resize_image.py:41-48"""
    height, width = image_size
    if mode == "keep_ratio":
        width = max(width, int(height / src_h * src_w / 32 + 0.5) * 32)
    if mode == "pad":
        width = min(width, max(int(height / src_h * src_w / 32 + 0.5) * 32, 32))
    return height, width


def resize_or_pad(img, image_size, mode):
    """resize_image.py:29-57 for modes resize / pad"""
    h, w = resized_width(mode, image_size, img.shape[0], img.shape[1])
    out = resize_bilinear_f32(img, h, w)
    if mode == "pad":
        canvas = np.zeros((image_size[0], image_size[1], 3), np.float32)
        canvas[:, :w, :] = out
        return canvas
    return out


def normalize(img):
    """normalize_image.py:13-16: in-place float32 array minus a float64 vector (computed in double, stored as float), then a
    float32 division; HWC -> CHW."""
    x = (img.astype(np.float64) - RGB_MEAN).astype(np.float32)
    x = x / np.float32(255.0)
    return np.ascontiguousarray(x.transpose(2, 0, 1))


def pack_label(text, lut, max_size=32):
    """concern/charsets.py:52-58 + make_recognition_label.py:22-31 -> (label int32 [max_size], length)"""
    label = np.zeros((max(max_size, len(text)),), np.int32)
    for i, ch in enumerate(text):
        label[i] = lut(ch)
    return label[:max_size], np.int32(min(len(text), max_size))
