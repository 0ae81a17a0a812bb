"""numpy restatement of the reference's model conversion (sfm/convert.py:26-96, save_depth_pose and
normalize_depth_for_display with cmap `binary`, then plt.imsave's byte conversion) — the checker of
particlesfm_b200.convert and csrc/convert.cu.

Two forms of the depth map:
  depth_maps_loop        the reference's loop over every keypoint of every image (convert.py:75-91), z from
                         np.matmul(K, R X + t) as it is written (z_order="reference") or in the kernel's order
  depth_maps             vectorised over each image's keypoints, z in the kernel's documented operation order:
                           z = ((R20 X + R21 Y) + R22 Z) + t2, every product and sum rounded (no FMA)
The display image (display_rgba) and the colormap (binary_lut) are recalled, not checked against matplotlib, which
is not a dependency: the table is the 256-entry one LinearSegmentedColormap builds for `binary`
(red = green = blue = ((0, 1, 1), (1, 0, 0))), the colormap indexes it with int(float32(n) * 256) (256 -> 255, NaN ->
the "bad" colour (0, 0, 0, 0)), and imsave stores (value * 255).astype(uint8) with alpha 255.
"""
import numpy as np


def qvec2rotmat(q):
    return np.array([
        [1 - 2 * q[2]**2 - 2 * q[3]**2, 2 * q[1] * q[2] - 2 * q[0] * q[3], 2 * q[3] * q[1] + 2 * q[0] * q[2]],
        [2 * q[1] * q[2] + 2 * q[0] * q[3], 1 - 2 * q[1]**2 - 2 * q[3]**2, 2 * q[2] * q[3] - 2 * q[0] * q[1]],
        [2 * q[3] * q[1] - 2 * q[0] * q[2], 2 * q[2] * q[3] + 2 * q[0] * q[1], 1 - 2 * q[1]**2 - 2 * q[2]**2]])


def binary_lut():
    """matplotlib's _create_lookup_table(256, ((0, 1, 1), (1, 0, 0))) times 255, truncated to uint8."""
    N = 256
    xind = (N - 1) * np.linspace(0, 1, N) ** 1.0
    # segment [0, 255]: y1 of its left end is 1, y0 of its right end is 0
    distance = (xind[1:-1] - 0.0) / (255.0 - 0.0)
    lut = np.concatenate([[1.0], distance * (0.0 - 1.0) + 1.0, [0.0]])
    return (np.clip(lut, 0.0, 1.0) * 255).astype(np.uint8)


def kernel_z(q, t, X):
    """z of the points X [n][3] in the kernel's operation order (numpy does not contract to FMA)."""
    r20 = 2 * q[3] * q[1] - 2 * q[0] * q[2]
    r21 = 2 * q[2] * q[3] + 2 * q[0] * q[1]
    r22 = 1 - 2 * (q[1] * q[1]) - 2 * (q[2] * q[2])
    return ((r20 * X[:, 0] + r21 * X[:, 1]) + r22 * X[:, 2]) + t[2]


def _pixel(xy, w, h):
    p = np.round(np.asarray(xy, np.float64).reshape(-1, 2)).astype(np.int32)
    p[:, 0] = np.clip(p[:, 0], 0, w - 1)
    p[:, 1] = np.clip(p[:, 1], 0, h - 1)
    return p


def _images(a):
    """(size (w, h), qvec, tvec, keypoints, point rows) per image of the flat arrays (see depth_maps)."""
    ids = np.asarray(a["point_ids"], np.int64)
    where = {int(p): r for r, p in enumerate(ids)}
    kp_ptr = np.asarray(a["keypoint_ptr"], np.int64)
    size = np.asarray(a["camera_size"], np.int64).reshape(-1, 2)
    for i in range(len(a["image_ids"])):
        lo, hi = kp_ptr[i], kp_ptr[i + 1]
        p3 = np.asarray(a["point3D_ids"], np.int64)[lo:hi]
        rows = np.array([where[int(p)] if p != -1 else -1 for p in p3], np.int64)
        c = int(a["image_camera"][i])
        yield (int(size[c, 0]), int(size[c, 1])), np.asarray(a["qvec"][i], np.float64), \
            np.asarray(a["tvec"][i], np.float64), np.asarray(a["keypoints"], np.float64)[lo:hi], rows


def depth_maps(a):
    """Vectorised depth maps of the flat arrays a (the keyword arguments of save_depth_pose_arrays)."""
    xyz = np.asarray(a["xyz"], np.float64).reshape(-1, 3)
    out = []
    for (w, h), q, t, xy, rows in _images(a):
        depth = np.zeros((h, w))
        m = rows >= 0
        if m.any():
            p = _pixel(xy[m], w, h)
            depth[p[:, 1], p[:, 0]] = kernel_z(q, t, xyz[rows[m]])        # fancy assignment: the last one wins
        out.append(depth)
    return out


def depth_maps_loop(a, z_order="reference"):
    """The reference's loop, one keypoint at a time; z from np.matmul(K, R @ X + t) or, z_order="kernel", kernel_z."""
    xyz = np.asarray(a["xyz"], np.float64).reshape(-1, 3)
    out = []
    for (w, h), q, t, xy, rows in _images(a):
        R, tt = qvec2rotmat(q), np.expand_dims(t, -1)
        pts, vxy = [], []
        for k in range(len(rows)):
            if rows[k] == -1:
                continue
            pts.append(xyz[rows[k]])
            vxy.append(xy[k])
        depth = np.zeros((h, w))
        if pts:
            P = np.transpose(np.array(pts))
            if z_order == "reference":
                K = np.array([[1.0, 0, 0.5], [0, 1.0, 0.5], [0, 0, 1]])
                z = np.transpose(np.matmul(K, np.matmul(R, P) + tt))[:, -1]
            else:
                z = kernel_z(q, t, P.T)
            p = _pixel(vxy, w, h)
            for k in range(len(z)):
                depth[p[k, 1], p[k, 0]] = z[k]
        out.append(depth)
    return out


def percentile_linear(values, q):
    """numpy's percentile, method "linear", restated: virtual index (n - 1) q / 100 and numpy's two-sided _lerp."""
    s = np.sort(np.asarray(values, np.float64))
    n = len(s)
    if n == 0:
        raise IndexError("percentile of no value")
    vi = (n - 1) * (q / 100)
    if vi >= n - 1:
        return s[-1]
    lo = int(np.floor(vi))
    g = vi - lo
    a, b = s[lo], s[lo + 1]
    d = b - a
    return b - d * (1 - g) if g >= 0.5 else a + d * g


def display_rgba(depth, lut=None):
    """normalize_depth_for_display(depth, 98, 'binary') as plt.imsave stores it: [h][w][4] uint8.  An image without
    a valid pixel raises IndexError, as np.percentile of an empty array does."""
    lut = binary_lut() if lut is None else lut
    valid = depth > 0
    with np.errstate(divide="ignore", invalid="ignore"):
        v = 1.0 / (depth + 1)
        z1 = np.percentile(v[valid], 98)
        z2 = np.percentile(v[valid], 2)
        n = np.clip((v - z2) / (z1 - z2), 0, 1)
        x = n.astype(np.float32) * np.float32(256)
        x[x == 256] = 255
        bad = np.isnan(x)
        idx = np.where(bad, 0, x).astype(int)
    grey = lut[idx]
    grey[bad] = 0
    out = np.empty(depth.shape + (4,), np.uint8)
    out[..., 0] = out[..., 1] = out[..., 2] = grey
    out[..., 3] = 255
    return out
