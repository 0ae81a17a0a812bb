"""The numpy restatement of the model conversion (oracle/convert_oracle.py) against itself and numpy: the vectorised
form equals the reference's keypoint loop, the known edge cases of the depth map and its display image, the percentile
against np.percentile, and the colormap and PNG writer of particlesfm_b200.convert."""
import zlib

import numpy as np
import pytest

from oracle import convert_oracle as co
from particlesfm_b200 import convert


def random_model(seed, sizes=((64, 48), (40, 56)), num_images=4, num_points=300, keypoints=(0, 400), dup=0.2):
    """Flat model arrays (save_depth_pose_arrays' keyword arguments): cameras SIMPLE_PINHOLE and SIMPLE_RADIAL of
    different sizes, points in front of and behind the cameras, keypoints inside and outside the image, some on x.5,
    some sharing a pixel, point ids not in row order."""
    rng = np.random.default_rng(seed)
    nc = len(sizes)
    point_ids = rng.permutation(np.arange(1, 3 * num_points))[:num_points] + 10
    xyz = rng.normal(size=(num_points, 3)) * [2, 2, 1] + [0, 0, 4]
    cams = rng.integers(0, nc, num_images)
    qvec = rng.normal(size=(num_images, 4)) * [1, 0.1, 0.1, 0.1] + [3, 0, 0, 0]
    qvec[0] *= 1.0001                                        # not unit: the rotation is not renormalised
    tvec = rng.normal(size=(num_images, 3)) * 0.2
    ptr, kps, p3 = [0], [], []
    for i in range(num_images):
        w, h = sizes[cams[i]]
        n = int(rng.integers(max(keypoints[0], 8), keypoints[1]))
        xy = rng.uniform([-3, -3], [w + 3, h + 3], size=(n, 2))
        half = rng.random(n) < 0.1
        xy[half] = np.floor(xy[half]) + 0.5
        d = rng.random(n) < dup
        xy[d] = xy[rng.integers(0, n, d.sum())]                # shared pixels
        ids = np.where(rng.random(n) < 0.7, point_ids[rng.integers(0, num_points, n)], -1)
        ids[0] = point_ids[0]
        kps.append(xy)
        p3.append(ids)
        ptr.append(ptr[-1] + n)
    return dict(camera_ids=np.arange(1, nc + 1), camera_size=np.array(sizes), cam_params=np.array(
        [[50.0 + c, sizes[c][0] / 2, sizes[c][1] / 2, 0.01 * c] for c in range(nc)]),
        image_ids=np.arange(1, num_images + 1), image_names=["frame_%03d.jpg" % i for i in range(num_images)],
        image_camera=cams, qvec=qvec, tvec=tvec, keypoint_ptr=np.array(ptr), keypoints=np.concatenate(kps),
        point3D_ids=np.concatenate(p3), point_ids=point_ids, xyz=xyz, camera_model=np.array([0, 2][:nc]))


def one_image(xy, z, w=8, h=6):
    """One image with identity pose: keypoint k at xy[k] sees a point of depth z[k] (None: no point)."""
    has = [v is not None for v in z]
    xyz = np.array([[0.0, 0.0, v] for v in z if v is not None]).reshape(-1, 3)
    return dict(camera_ids=[1], camera_size=np.array([[w, h]]), cam_params=np.array([[10.0, 4, 3]]), image_ids=[1],
                image_names=["a.png"], image_camera=[0], qvec=np.array([[1.0, 0, 0, 0]]), tvec=np.zeros((1, 3)),
                keypoint_ptr=np.array([0, len(z)]), keypoints=np.array(xy, np.float64).reshape(-1, 2),
                point3D_ids=np.where(has, np.cumsum(has), -1), point_ids=np.arange(1, sum(has) + 1), xyz=xyz)


@pytest.mark.parametrize("seed", range(6))
def test_vectorised_form_equals_the_keypoint_loop(seed):
    a = random_model(seed)
    vec, loop_k, loop_r = co.depth_maps(a), co.depth_maps_loop(a, "kernel"), co.depth_maps_loop(a)
    # the reference's BLAS sum has its own order: a few rounding errors of the largest term (|R| |X| with |q| ~ 3)
    scale = 16 * np.abs(a["qvec"]).max() ** 2 * (np.abs(a["xyz"]).max() + 1)
    for d, k, r in zip(vec, loop_k, loop_r):
        assert np.array_equal(d, k)
        assert np.array_equal(d != 0, r != 0)
        assert np.all(np.abs(d - r) <= 4 * np.finfo(float).eps * scale)


def test_last_keypoint_wins_a_shared_pixel():
    d = co.depth_maps(one_image([[2.2, 1.1], [1.9, 0.8], [2.4, 1.4], [5, 5]], [3.0, 2.0, 4.0, 1.0]))[0]
    assert d[1, 2] == 4.0 and d[5, 5] == 1.0 and np.count_nonzero(d) == 2
    d = co.depth_maps(one_image([[2.2, 1.1], [1.9, 0.8], [2, 1]], [3.0, 2.0, None]))[0]
    assert d[1, 2] == 2.0                       # a keypoint without a point claims nothing


def test_half_to_even_rounding_and_clipping():
    d = co.depth_maps(one_image([[2.5, 0.5], [3.5, 1.5], [-7.2, 2.0], [20.0, 40.0], [-0.5, 5.5]],
                                [1.0, 2.0, 3.0, 4.0, 5.0]))[0]
    assert d[0, 2] == 1.0 and d[2, 4] == 2.0 and d[2, 0] == 3.0 and d[5, 7] == 4.0
    assert d[5, 0] == 5.0 and np.count_nonzero(d) == 5      # 5.5 -> 6 -> clipped to 5; -0.5 -> -0 -> 0


def test_negative_depth_and_minus_one_are_written_and_displayed():
    d = co.depth_maps(one_image([[0, 0], [1, 0], [2, 0], [3, 0], [4, 0]], [-2.0, -1.0, 1.0, 2.0, -0.5]))[0]
    assert d[0, 0] == -2.0 and d[0, 1] == -1.0 and d[0, 4] == -0.5
    lut = co.binary_lut()
    rgba = co.display_rgba(d, lut)
    # v: -1 (clipped to 0), inf (1), then 1/2 and 1/3 between the percentiles, 2 (1); empty pixels have v = 1
    assert rgba[0, 0, 0] == lut[0] and rgba[0, 1, 0] == lut[255] and rgba[0, 4, 0] == lut[255]
    assert rgba[1, 1, 0] == lut[255] and (rgba[..., 3] == 255).all()


def test_equal_valid_values_take_the_bad_colour():
    d = co.depth_maps(one_image([[0, 0], [3, 2], [5, 5]], [2.0, 2.0, 2.0]))[0]
    rgba = co.display_rgba(d)
    assert (rgba[d > 0, :3] == 0).all()                      # 0 / 0: NaN -> black
    assert (rgba[d == 0, :3] == co.binary_lut()[255]).all()  # 1 / 0: inf -> 1
    assert (rgba[..., 3] == 255).all()


def test_an_image_without_a_valid_pixel_raises_index_error():
    d = co.depth_maps(one_image([[0, 0], [1, 1]], [-3.0, 0.0]))[0]
    with pytest.raises(IndexError):
        co.display_rgba(d)


@pytest.mark.parametrize("seed", range(4))
def test_percentile_restatement_equals_numpy(seed):
    rng = np.random.default_rng(seed)
    for n in list(range(1, 60)) + [101, 1000, 4097]:
        v = 1 / (rng.exponential(3, n) + 1)
        if n > 5:
            v[: n // 4] = v[0]                               # ties
        for q in (98, 2, 50, 0, 100):
            assert co.percentile_linear(v, q) == np.percentile(v, q), (n, q)


def test_binary_lut_of_the_product_equals_the_restatement():
    lut = convert.binary_lut()
    assert lut.dtype == np.uint8 and lut.shape == (256,)
    assert np.array_equal(lut, co.binary_lut())
    assert lut[0] == 255 and lut[255] == 0 and np.all(np.diff(lut.astype(int)) <= 0)


def read_png_rgba(path):
    """Pixels of an RGBA8 PNG whose rows all use filter 0 (what convert.write_png_rgba writes)."""
    buf = open(path, "rb").read()
    assert buf[:8] == b"\x89PNG\r\n\x1a\n"
    o, idat, w, h = 8, b"", None, None
    while o < len(buf):
        n = int.from_bytes(buf[o:o + 4], "big")
        tag, data = buf[o + 4:o + 8], buf[o + 8:o + 8 + n]
        assert zlib.crc32(tag + data) & 0xffffffff == int.from_bytes(buf[o + 8 + n:o + 12 + n], "big")
        if tag == b"IHDR":
            w, h = int.from_bytes(data[:4], "big"), int.from_bytes(data[4:8], "big")
            assert data[8:] == bytes([8, 6, 0, 0, 0])
        elif tag == b"IDAT":
            idat += data
        o += 12 + n
    raw = np.frombuffer(zlib.decompress(idat), np.uint8).reshape(h, 1 + 4 * w)
    assert (raw[:, 0] == 0).all()
    return raw[:, 1:].reshape(h, w, 4)


def test_png_writer_round_trips(tmp_path):
    rgba = np.random.default_rng(1).integers(0, 256, (7, 13, 4)).astype(np.uint8)
    convert.write_png_rgba(str(tmp_path / "x.png"), rgba)
    assert np.array_equal(read_png_rgba(str(tmp_path / "x.png")), rgba)
