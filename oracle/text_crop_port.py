"""Plain restatement of the reference's text crop on cv2: concern/cv.py's min_area_rect and ImageCropper.crop
(data/crop_file_dataset.py:85-124) with ResizeImage's "resize" and "pad" modes and NormalizeImage's arithmetic.

One change makes it run on current cv2: warpPerspective's dsize is (int(w), int(h)) -- the reference passes numpy float32
sides, which cv2 4.x refuses ("Can't parse 'dsize'").  int() truncates; when either side truncates to 0 cv2 takes the
source's size for the crop (DESIGN §7)."""
import cv2
import numpy as np

RGB_MEAN = np.array([122.67891434, 116.66876762, 104.00698793])


def min_area_rect(poly):
    """cv2.minAreaRect of the float32 polygon, then: angle < -45 -> angle + 180; else the sides swap and angle + 90;
    cv2.boxPoints of the result ([4, 2] float32)"""
    (cx, cy), (w, h), angle = cv2.minAreaRect(np.asarray(poly, np.float32))
    if angle < -45:
        rect = ((cx, cy), (w, h), angle + 180)
    else:
        rect = ((cx, cy), (h, w), angle + 90)
    return cv2.boxPoints(rect)


def crop_geometry(poly):
    """(box [4, 2] float32, w, h float32, P float64 [3, 3], (int(w), int(h)))"""
    box = min_area_rect(poly)
    w = np.linalg.norm(box[1] - box[0])
    h = np.linalg.norm(box[2] - box[1])
    dst = np.array([(0, 0), (w, 0), (w, h), (0, h)], np.float32)
    P = cv2.getPerspectiveTransform(box.astype(np.float32), dst)
    return box, w, h, P, (int(w), int(h))


def ensure_horizontal(image):
    h, w = image.shape[:2]
    if h > w * 1.5:
        image = np.flip(np.swapaxes(image, 0, 1), 0)
    return image


def resized_width(mode, image_size, src_h, src_w):
    height, width = image_size
    if mode == "pad":
        width = min(width, max(int(height / src_h * src_w / 32 + 0.5) * 32, 32))
    elif mode != "resize":
        raise ValueError("mode %r" % (mode,))
    return width


def resize(image, image_size, mode):
    height = image_size[0]
    width = resized_width(mode, image_size, *image.shape[:2])
    out = cv2.resize(image, (width, height))
    if mode == "pad":
        canvas = np.zeros((*image_size, 3), np.float32)
        canvas[:, :width, :] = out
        out = canvas
    return out


def warp(image, poly):
    """The crop as float32 (the warp of the source through the min-area rectangle)"""
    _, _, _, P, size = crop_geometry(poly)
    return cv2.warpPerspective(image, P, size).astype(np.float32)


def finish(cropped, image_size, mode):
    """ensure_horizontal, ResizeImage and NormalizeImage of a float32 crop"""
    out = resize(ensure_horizontal(cropped), image_size, mode)
    out -= RGB_MEAN
    out /= 255.
    return out


def crop(image, poly, image_size=(64, 512), mode="resize"):
    """ImageCropper(image_size, mode).crop(image, poly): HWC float32 [image_size[0], image_size[1], 3]"""
    return finish(warp(image, poly), image_size, mode)


def crop_with_matrix(image, P, dsize, image_size=(64, 512), mode="resize"):
    """The same crop from a given perspective matrix and dsize (the steps after min_area_rect and getPerspectiveTransform)"""
    return finish(cv2.warpPerspective(image, P, tuple(int(v) for v in dsize)).astype(np.float32), image_size, mode)
