"""The restated colour extraction (oracle/colors_oracle.py) on hand-computed cases, and its literal loop against its
vectorised form."""
import numpy as np
import pytest

from oracle import colors_oracle as co


def ramp(w=4, h=3):
    """img[r][c][ch] = 40 r + 10 c + ch: every pixel and channel distinct."""
    r, c, ch = np.meshgrid(np.arange(h), np.arange(w), np.arange(3), indexing="ij")
    return (40 * r + 10 * c + ch).astype(np.uint8)


def test_integer_coordinates_return_the_pixel():
    img = ramp()
    for x, y in ((0, 1), (1, 1), (2, 2), (1, 2)):
        assert np.array_equal(co.interpolate_bilinear(img, float(x), float(y)), img[y, x].astype(np.float32)), (x, y)


def test_fractional_coordinates_by_hand():
    img = ramp()
    # between rows 1 and 2 and a quarter of the way from column 0 to 1: the mean of 40 + 2.5 and 80 + 2.5, per channel
    assert np.array_equal(co.interpolate_bilinear(img, 0.25, 1.5), np.float32([62.5, 63.5, 64.5]))
    # x = 2.75, y = 1.125: row 1 + 1/8 of the way to row 2, column 2 + 3/4 of the way to column 3
    assert np.array_equal(co.interpolate_bilinear(img, 2.75, 1.125), np.float32([40 + 5 + 27.5, 40 + 5 + 28.5, 40 + 5 + 29.5]))


def test_the_asymmetric_edges():
    img = ramp()
    h, w = img.shape[:2]
    # at integer x, the last column is rejected (x1 = w) and column 0 is accepted
    assert co.interpolate_bilinear(img, float(w - 1), 1.0) is None
    assert np.array_equal(co.interpolate_bilinear(img, 0.0, 1.0), img[1, 0].astype(np.float32))
    # at integer y, row 0 is rejected (inv_y = h - 1, y1 = h) and the last row is accepted
    assert co.interpolate_bilinear(img, 1.0, 0.0) is None
    assert np.array_equal(co.interpolate_bilinear(img, 1.0, float(h - 1)), img[h - 1, 1].astype(np.float32))
    # just outside the accepted ranges, and coordinates that are not numbers
    for x, y in ((-1e-9, 1.0), (w - 2 + 1e-9 + 1, 1.0), (1.0, h - 1 + 1e-9), (1.0, 1e-300 * 0.0 - 1e-12),
                 (np.nan, 1.0), (1.0, np.nan), (1e300, 1.0), (1.0, -1e300)):
        assert co.interpolate_bilinear(img, x, y) is None, (x, y)


def _obs(img_xy_rows):
    """keypoint_ptr, keypoints and rows of per-image lists of (X, Y, row) in COLMAP's convention (pixel centre 0.5)."""
    ptr, kp, rows = [0], [], []
    for obs in img_xy_rows:
        for X, Y, r in obs:
            kp.append([X, Y])
            rows.append(r)
        ptr.append(len(kp))
    return np.array(ptr), np.array(kp, np.float64).reshape(-1, 2), np.array(rows)


@pytest.mark.parametrize("form", ["loop", "vectorised"])
def test_round_half_away_no_sample_and_a_missing_image(form):
    f = co.extract_colors_loop if form == "loop" else co.extract_colors
    a = np.zeros((3, 4, 3), np.uint8)
    a[1, 1] = (2, 200, 7)
    b = np.zeros((3, 4, 3), np.uint8)
    b[1, 1] = (3, 201, 8)
    c = np.full((3, 4, 3), 90, np.uint8)
    # point 0: 2 + 3 = k + 0.5 with k = 2 (rounds to 3, not to the even 2), 200.5 -> 201, 7.5 -> 8
    # point 1: only observed outside the accepted ranges -> black; point 2: never observed -> black
    # point 3: seen in the missing image and in c -> c's colour only
    ptr, kp, rows = _obs([[(1.5, 1.5, 0), (3.5, 1.5, 1)], [(1.5, 1.5, 0), (1.5, 0.5, 1)],
                          [(1.5, 1.5, 3)], [(2.0, 2.0, 3)]])
    rgb = f([a, b, None, c], ptr, kp, rows, 4)
    assert rgb.tolist() == [[3, 201, 8], [0, 0, 0], [0, 0, 0], [90, 90, 90]]
    assert co.round_half_away(2.5) == 3 and co.round_half_away(2.4999999999999996) == 2 and co.round_half_away(0.5) == 1


def random_images(rng, n, lo=5, hi=40):
    return [rng.integers(0, 256, (int(rng.integers(lo, hi)), int(rng.integers(lo, hi)), 3), dtype=np.uint8)
            for _ in range(n)]


def edge_keypoints(w, h):
    """Every edge case of the interpolation in COLMAP coordinates (X = x + 0.5): integer and fractional positions at
    and beside the four edges, negative, NaN and huge coordinates."""
    xs = [0.5, 1.5, w - 1.5, w - 0.5, w - 1.0, 0.0, 0.499, 0.75, w / 2 + 0.123, -3.0, np.nan, 1e300]
    ys = [0.5, 1.5, h - 1.5, h - 0.5, h - 1.0, 0.0, 0.499, 1.25, h / 2 + 0.377, -2.0, np.nan, -1e300]
    return np.array([[x, y] for x in xs for y in ys], np.float64)


def random_model(rng, images, num_points, per_image=60, edges=True):
    """keypoint_ptr, keypoints and point rows over the images: random positions around and inside each image, the
    edge cases, keypoints without a point, points observed by many images and points observed by none."""
    ptr, kps, rows = [0], [], []
    for img in images:
        h, w = img.shape[:2]
        kp = np.stack([rng.uniform(-2, w + 2, per_image), rng.uniform(-2, h + 2, per_image)], 1)
        if edges:
            kp = np.concatenate([kp, edge_keypoints(w, h)])
        r = rng.integers(-1, num_points - 3, len(kp))          # the last three points are never observed
        kps.append(kp)
        rows.append(r)
        ptr.append(ptr[-1] + len(kp))
    return np.array(ptr, np.int64), np.concatenate(kps), np.concatenate(rows).astype(np.int32)


def test_literal_loop_equals_the_vectorised_form():
    rng = np.random.default_rng(11)
    images = random_images(rng, 7)
    images[3] = None
    ptr, kp, rows = random_model(rng, [np.zeros((9, 9, 3)) if i is None else i for i in images], 50)
    loop = co.extract_colors_loop(images, ptr, kp, rows, 50)
    vec = co.extract_colors(images, ptr, kp, rows, 50)
    assert np.array_equal(loop, vec)
    assert (loop[:-3] > 0).any(axis=1).sum() > 30 and not loop[-3:].any()
