"""Restatement of the reference's colour extraction (Reconstruction::ExtractColorsForAllImages, reference
base/reconstruction.cc:1250-1300) — the checker of particlesfm_b200.colors and csrc/colors.cu.

Two forms, with the same summation order (ascending image index, then keypoint index; the reference's order over
reg_image_ids_ is not defined):
  extract_colors_loop    the reference loop, literally: images in ascending index, a dict of per-point sums and counts,
                         Bitmap::InterpolateBilinear on FreeImage's bottom-up scanlines, emulated by indexing the
                         vertically flipped image with the scanline number, in Python doubles with a np.float32 store
  extract_colors         vectorised over each image's observations; np.add.at adds in index order
Both take the decoded images as top-down [h][w][3] uint8 arrays (None: the image could not be read).

Bitmap::InterpolateBilinear and Bitmap::Read(as_rgb = true) are COLMAP 3.8 code the reference does not vendor; they are
recalled, not pinned to a source line (RECALLED; csrc/colors_recalled.cuh restates the same function):
  inv_y = h - 1 - y, x0 = floor(x), y0 = floor(inv_y), x1 = x0 + 1, y1 = y0 + 1; no sample if x0 < 0, x1 >= w, y0 < 0
  or y1 >= h; dx = x - x0, dy = inv_y - y0, dx_1 = 1 - dx, dy_1 = 1 - dy;
  c = dx_1 dy_1 p00 + dx dy_1 p01 + dx_1 dy p10 + dx dy p11 (double, left to right, stored as float), p00 / p01 at
  columns x0 / x1 of scanline y0, p10 / p11 of scanline y1.
The bounds are tested on the floors as doubles, so NaN and coordinates beyond int's range are no sample.  Read converts
to 24-bit RGB: grey replicated, alpha dropped (not composited), palettes expanded — what Pillow's convert("RGB") does
for modes RGB, RGBA, L, LA and P.
"""
import math

import numpy as np

RECALLED = {
    "pixel_centre": 0.5,        # ExtractColorsForAllImages samples at (X - 0.5, Y - 0.5)
    "modes": ("RGB", "RGBA", "L", "LA", "P"),
}


def read_image(path):
    """Bitmap::Read(path, as_rgb = true) by Pillow: [h][w][3] uint8, or None when the file cannot be read."""
    from PIL import Image
    try:
        with Image.open(path) as im:
            if im.mode not in RECALLED["modes"]:
                raise ValueError(f"{path}: mode {im.mode}")
            return np.asarray(im.convert("RGB"))
    except OSError:
        return None


def interpolate_bilinear(img, x, y):
    """Bitmap::InterpolateBilinear(x, y) of the top-down image img: np.float32 [3], or None (no sample)."""
    h, w = img.shape[:2]
    bottom_up = img[::-1]                    # FreeImage's scanline s is top-down row h - 1 - s
    inv_y = (h - 1) - y
    fx, fy = np.floor(x), np.floor(inv_y)
    if not (fx >= 0 and fx <= w - 2 and fy >= 0 and fy <= h - 2):
        return None
    x0, y0 = int(fx), int(fy)
    x1, y1 = x0 + 1, y0 + 1
    dx, dy = x - x0, inv_y - y0
    dx_1, dy_1 = 1 - dx, 1 - dy
    line0, line1 = bottom_up[y0], bottom_up[y1]
    out = np.zeros(3, np.float32)
    for c in range(3):
        out[c] = np.float32(dx_1 * dy_1 * float(line0[x0][c]) + dx * dy_1 * float(line0[x1][c])
                            + dx_1 * dy * float(line1[x0][c]) + dx * dy * float(line1[x1][c]))
    return out


def round_half_away(v):
    """std::round of a non-negative double."""
    r = math.floor(v)
    return r + 1 if v - r >= 0.5 else r


def extract_colors_loop(images, keypoint_ptr, keypoints, point_of_keypoint, num_points):
    """The reference loop: rgb [num_points][3] uint8.  point_of_keypoint: point row of each keypoint, -1: none."""
    sums, counts = {}, {}
    for i, img in enumerate(images):
        if img is None:
            continue
        for k in range(int(keypoint_ptr[i]), int(keypoint_ptr[i + 1])):
            p = int(point_of_keypoint[k])
            if p < 0:
                continue
            x, y = float(keypoints[k][0]), float(keypoints[k][1])
            color = interpolate_bilinear(img, x - RECALLED["pixel_centre"], y - RECALLED["pixel_centre"])
            if color is None:
                continue
            if p in sums:
                s = sums[p]
                sums[p] = [s[0] + float(color[0]), s[1] + float(color[1]), s[2] + float(color[2])]
                counts[p] += 1
            else:
                sums[p] = [float(color[0]), float(color[1]), float(color[2])]
                counts[p] = 1
    rgb = np.zeros((num_points, 3), np.uint8)
    for p in range(num_points):
        if p in sums:
            rgb[p] = [round_half_away(s / counts[p]) for s in sums[p]]
    return rgb


def sample_image(img, xy):
    """InterpolateBilinear at (x - 0.5, y - 0.5) of every row of xy [n][2]: (ok [n] bool, colour [n][3] float32)."""
    h, w = img.shape[:2]
    x = xy[:, 0] - RECALLED["pixel_centre"]
    inv_y = (h - 1) - (xy[:, 1] - RECALLED["pixel_centre"])
    fx, fy = np.floor(x), np.floor(inv_y)
    with np.errstate(invalid="ignore"):
        ok = (fx >= 0) & (fx <= w - 2) & (fy >= 0) & (fy <= h - 2)
    x0, y0 = fx[ok].astype(np.int64), fy[ok].astype(np.int64)
    dx, dy = (x[ok] - x0)[:, None], (inv_y[ok] - y0)[:, None]
    dx_1, dy_1 = 1 - dx, 1 - dy
    r0, r1 = h - 1 - y0, h - 2 - y0          # top-down rows of scanlines y0 and y1
    f = img.astype(np.float64)
    c = dx_1 * dy_1 * f[r0, x0] + dx * dy_1 * f[r0, x0 + 1] + dx_1 * dy * f[r1, x0] + dx * dy * f[r1, x0 + 1]
    colour = np.zeros((len(xy), 3), np.float32)
    colour[ok] = c.astype(np.float32)
    return ok, colour


def extract_colors(images, keypoint_ptr, keypoints, point_of_keypoint, num_points):
    """Vectorised form of extract_colors_loop, the same sums in the same order."""
    keypoints = np.asarray(keypoints, np.float64).reshape(-1, 2)
    rows = np.asarray(point_of_keypoint, np.int64)
    sums = np.zeros((num_points, 3))
    counts = np.zeros(num_points, np.int64)
    for i, img in enumerate(images):
        if img is None:
            continue
        lo, hi = int(keypoint_ptr[i]), int(keypoint_ptr[i + 1])
        has = rows[lo:hi] >= 0
        ok, colour = sample_image(img, keypoints[lo:hi][has])
        p = rows[lo:hi][has][ok]
        np.add.at(sums, p, colour[ok].astype(np.float64))
        np.add.at(counts, p, 1)
    rgb = np.zeros((num_points, 3), np.uint8)
    m = counts > 0
    v = sums[m] / counts[m][:, None]
    r = np.floor(v)
    rgb[m] = (r + (v - r >= 0.5)).astype(np.uint8)
    return rgb
