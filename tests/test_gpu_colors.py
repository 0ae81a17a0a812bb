"""The colour extraction on the device (csrc/colors.cu, particlesfm_b200.colors) against the restated reference loop
(oracle/colors_oracle.py): colours bit for bit on PNGs of every accepted mode and on JPEGs given the same decoded
pixels, in the global mapper and in the color_extractor command."""
import os
import struct

import numpy as np
import pytest
from PIL import Image

from oracle import colors_oracle as co
from particlesfm_b200 import colmap_io, colors, global_mapper as gm
from test_gpu_global_mapper import H, W, _scene_db
from test_oracle_colors import random_images, random_model

pytestmark = pytest.mark.gpu


def _save(img, path, mode):
    """img (RGB8) in Pillow mode `mode`; the path's extension picks the format."""
    os.makedirs(os.path.dirname(path), exist_ok=True)
    im = Image.fromarray(img)
    if mode == "RGBA":
        im = Image.fromarray(np.concatenate([img, img[..., :1]], -1), "RGBA")
    elif mode == "L":
        im = im.convert("L")
    elif mode == "LA":
        im = Image.fromarray(np.stack([img[..., 0], img[..., 1]], -1), "LA")
    elif mode == "P":
        im = im.quantize(64)
    im.save(path)
    with Image.open(path) as check:
        assert check.mode == mode, (path, check.mode)


def _images(tmp_path, rng, n, ext, modes):
    names = []
    for i, img in enumerate(random_images(rng, n, 6, 48)):
        name = os.path.join("sub%d" % (i % 2), "f%03d%s" % (i, ext))
        _save(img, str(tmp_path / name), modes[i % len(modes)])
        names.append(name)
    return names


@pytest.mark.parametrize("budget", [1 << 14, 256 << 20])
def test_png_modes_equal_the_oracle(gpu, tmp_path, budget):
    rng = np.random.default_rng(5)
    names = _images(tmp_path, rng, 15, ".png", ["RGB", "RGBA", "L", "LA", "P"])
    (tmp_path / "broken.png").write_bytes(b"\x89PNG\r\n\x1a\n not a png")
    (tmp_path / "trunc.png").write_bytes((tmp_path / names[0]).read_bytes()[:200])     # its header reads, its data not
    names[4:4] = ["missing.png", "broken.png"]
    names[9:9] = ["trunc.png"]
    decoded = [co.read_image(str(tmp_path / n)) for n in names]
    P = 300
    ptr, kp, rows = random_model(rng, [np.zeros((9, 9, 3)) if d is None else d for d in decoded], P)
    rgb, rep = colors.extract_colors_for_all_images(str(tmp_path), names, ptr, kp, rows, P, memory_budget=budget,
                                                    verbose=False)
    ref = co.extract_colors(decoded, ptr, kp, rows, P)
    assert np.array_equal(rgb, ref)
    assert np.array_equal(rgb, co.extract_colors_loop(decoded, ptr, kp, rows, P))
    assert rep.unread == ["missing.png", "broken.png", "trunc.png"] and rep.images == 15
    assert rep.num_observations == int((rows >= 0).sum())
    assert rep.num_batches >= (3 if budget < 1 << 20 else 2)      # the unread images split the run of images
    assert (rgb[:-3] > 0).any(axis=1).sum() > 200 and not rgb[-3:].any()
    # two calls give the same bytes
    again, _ = colors.extract_colors_for_all_images(str(tmp_path), names, ptr, kp, rows, P, memory_budget=budget,
                                                    verbose=False)
    assert np.array_equal(again, rgb)


def test_jpeg_equals_the_oracle_on_the_same_pixels(gpu, tmp_path, capsys):
    rng = np.random.default_rng(6)
    names = _images(tmp_path, rng, 12, ".jpg", ["RGB", "L"]) + ["nothing/here.jpg"]
    decoded = [co.read_image(str(tmp_path / n)) for n in names]
    P = 200
    ptr, kp, rows = random_model(rng, [np.zeros((9, 9, 3)) if d is None else d for d in decoded], P)
    rgb, rep = colors.extract_colors_for_all_images(str(tmp_path), names, ptr, kp, rows, P, memory_budget=1 << 13)
    assert np.array_equal(rgb, co.extract_colors(decoded, ptr, kp, rows, P))
    assert rep.unread == ["nothing/here.jpg"] and rep.num_batches >= 3
    out = capsys.readouterr().out
    assert out == "Could not read image nothing/here.jpg at path %s.\n" % os.path.join(str(tmp_path), "nothing/here.jpg")


def test_no_image_and_no_observation(gpu, tmp_path):
    rgb, rep = colors.extract_colors_for_all_images(str(tmp_path), [], np.zeros(1, np.int64), np.zeros((0, 2)),
                                                    np.zeros(0, np.int32), 5, verbose=False)
    assert rgb.shape == (5, 3) and not rgb.any() and rep.num_batches == 0


def _frames(path, n):
    """Rendered frames of the helix scene: a smooth colour field per frame, with seeded noise, W x H RGB PNGs."""
    os.makedirs(path, exist_ok=True)
    yy, xx = np.mgrid[0:H, 0:W]
    rng = np.random.default_rng(3)
    for i in range(n):
        f = np.stack([127 + 120 * np.sin(xx / (37.0 + i) + c) * np.cos(yy / 23.0 - c * i) for c in range(3)], -1)
        img = np.clip(f + rng.normal(0, 6, f.shape), 0, 255).astype(np.uint8)
        Image.fromarray(img).save(os.path.join(path, "%05d.png" % i))


def _model_colors_oracle(model_dir, image_dir):
    m = colmap_io.read_model(model_dir)
    ims, pts = list(m.images.values()), list(m.points3D.values())
    ptr = np.concatenate([[0], np.cumsum([len(im.xys) for im in ims])]).astype(np.int64)
    rows = colors.point_rows(np.concatenate([im.point3D_ids for im in ims]), [p.point3D_id for p in pts])
    decoded = [co.read_image(os.path.join(image_dir, im.name)) for im in ims]
    ref = co.extract_colors(decoded, ptr, np.concatenate([im.xys for im in ims]), rows, len(pts))
    return np.array([p.rgb for p in pts]), ref


def _rgb_offsets(points3D_bin):
    """Byte offsets of every point's rgb in a points3D.bin."""
    buf = open(points3D_bin, "rb").read()
    (n,), o, out = struct.unpack_from("<Q", buf, 0), 8, []
    for _ in range(n):
        out.append(o + 32)
        (l,) = struct.unpack_from("<Q", buf, o + 43)
        o += 51 + 8 * l
    assert o == len(buf)
    return np.array(out, np.int64)


@pytest.fixture(scope="module")
def mapped(tmp_path_factory):
    d = tmp_path_factory.mktemp("colors_mapper")
    db = str(d / "database.db")
    _scene_db(db)
    _frames(str(d / "images"), 10)
    o = gm.GlobalMapperOptions(ba_refine_principal_point=False, ba_refine_extra_params=False)
    plain = gm.global_mapper(db, str(d / "plain"), o)
    coloured = gm.global_mapper(db, str(d / "coloured"), o, image_path=str(d / "images"))
    return d, plain, coloured


def test_mapper_colours_equal_the_oracle(gpu, mapped):
    d, plain, coloured = mapped
    assert plain.success and coloured.success
    got, ref = _model_colors_oracle(coloured.output, str(d / "images"))
    assert np.array_equal(got, ref) and (got > 0).any(axis=1).mean() > 0.9
    summary = [s for n, _, s in coloured.stages if n == "colors"][0]
    assert summary["unread"] == [] and coloured.seconds("colors") > 0
    assert "ExtractColors" not in coloured.not_run and len(coloured.not_run) == 3
    assert set(plain.not_run) == set(gm.NOT_RUN) and "colors" not in [n for n, _, _ in plain.stages]
    # the rest of the model is the run without images: ids, names, tracks and observations exactly; the bundle
    # adjustment's reductions are not in a fixed order (DESIGN.md §3.2), so poses and points agree to rounding
    a, b = colmap_io.read_model(plain.output), colmap_io.read_model(coloured.output)
    assert list(a.cameras) == list(b.cameras) and list(a.images) == list(b.images) and list(a.points3D) == list(b.points3D)
    for i in a.images:
        x, y = a.images[i], b.images[i]
        assert x.name == y.name and np.array_equal(x.point3D_ids, y.point3D_ids) and np.array_equal(x.xys, y.xys)
        assert np.abs(x.tvec - y.tvec).max() <= 1e-9 * max(np.abs(x.tvec).max(), 1.0)
    for p in a.points3D:
        x, y = a.points3D[p], b.points3D[p]
        assert not x.rgb.any() and np.array_equal(x.image_ids, y.image_ids) and np.array_equal(x.point2D_idxs, y.point2D_idxs)
        assert np.abs(x.xyz - y.xyz).max() <= 1e-9 * max(np.abs(x.xyz).max(), 1.0)


def test_mapper_without_readable_images_writes_black_points(gpu, mapped, capsys):
    d, plain, _ = mapped
    out = str(d / "unread")
    assert gm.main(["--database_path", str(d / "database.db"), "--image_path", str(d / "nowhere"), "--output_path", out,
                    "--GlobalMapper.ba_refine_principal_point", "0", "--GlobalMapper.ba_refine_extra_params", "0"]) == 0
    text = capsys.readouterr().out
    m = colmap_io.read_model(os.path.join(out, "0"))
    for im in m.images.values():
        assert "Could not read image %s at path %s." % (im.name, os.path.join(str(d / "nowhere"), im.name)) in text
    assert not np.array([p.rgb for p in m.points3D.values()]).any()
    assert "not run: CompleteAndMergeTracks, Retriangulate, FilterImages)" in text
    # --GlobalMapper.extract_colors 0 keeps the step off
    assert gm.main(["--database_path", str(d / "database.db"), "--image_path", str(d / "images"), "--output_path",
                    str(d / "off"), "--GlobalMapper.extract_colors", "0", "--quiet"]) == 0
    m = colmap_io.read_model(os.path.join(str(d / "off"), "0"))
    assert not np.array([p.rgb for p in m.points3D.values()]).any()


def test_color_extractor_changes_only_rgb_bytes(gpu, mapped):
    d, plain, _ = mapped
    out = str(d / "extracted")
    assert colors.main(["--image_path", str(d / "images"), "--input_path", plain.output, "--output_path", out]) == 0
    for n in ("cameras.bin", "images.bin"):
        assert open(os.path.join(plain.output, n), "rb").read() == open(os.path.join(out, n), "rb").read(), n
    a = np.frombuffer(open(os.path.join(plain.output, "points3D.bin"), "rb").read(), np.uint8)
    b = np.frombuffer(open(os.path.join(out, "points3D.bin"), "rb").read(), np.uint8)
    assert len(a) == len(b)
    rgb = (_rgb_offsets(os.path.join(out, "points3D.bin"))[:, None] + np.arange(3)).reshape(-1)
    keep = np.ones(len(a), bool)
    keep[rgb] = False
    assert np.array_equal(a[keep], b[keep]) and not a[rgb].any() and b[rgb].any()
    got, ref = _model_colors_oracle(out, str(d / "images"))
    assert np.array_equal(got, ref)
