"""The SfM driver's host side (particlesfm_b200.sfm): the database schema against the reference's create_empty_db, the
feature_importer rules on PNG directories, every refusal before any library call, and the command line's flags."""
import json
import os
import sqlite3
import sys

import numpy as np
import pytest
from PIL import Image

from particlesfm_b200 import _lib, sfm

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
from make_sfm_golden import schema_rows  # noqa: E402


def _frames(path, sizes, fmt="png", exif=None):
    os.makedirs(path, exist_ok=True)
    names = []
    for i, (w, h) in enumerate(sizes):
        names.append("%05d.%s" % (i, fmt))
        img = Image.fromarray(np.full((h, w, 3), 10 * i, np.uint8))
        img.save(os.path.join(path, names[-1]), **({"exif": exif} if exif is not None and i == len(sizes) - 1 else {}))
    return names


def _tracks(num_frames, n=30, seed=0):
    rng = np.random.default_rng(seed)
    out = {}
    for k in range(n):
        f0 = int(rng.integers(0, num_frames - 2))
        frames = list(range(f0, min(num_frames, f0 + 3)))
        out[k] = {"frame_ids": frames, "locations": rng.random((len(frames), 2)) * 30, "labels": [0] * len(frames)}
    return out


@pytest.fixture
def no_library(monkeypatch):
    def refuse():
        raise AssertionError("the library was called")
    monkeypatch.setattr(_lib, "lib", refuse)


def test_schema_matches_reference_create_empty_db(tmp_path):
    with open(os.path.join(HERE, "golden", "sfm_schema.json")) as f:
        ref = json.load(f)
    con = sqlite3.connect(str(tmp_path / "database.db"))
    con.executescript(sfm.SCHEMA)
    got = json.loads(json.dumps(schema_rows(con)))
    con.close()
    assert got == ref


def test_importer_rules(tmp_path):
    img = tmp_path / "images"
    names = _frames(str(img), [(40, 30)] * 3)
    os.rename(img / names[0], img / "zz.png")              # ids follow the sorted names, not the creation order
    images = sfm.read_image_set(str(img))
    assert images.names == sorted(names[1:] + ["zz.png"])
    assert images.image_ids.tolist() == [1, 2, 3]
    assert (images.width, images.height) == (40, 30)
    assert images.camera.tolist() == [1.2 * 40, 20.0, 15.0]
    con = sqlite3.connect(str(tmp_path / "database.db"))
    sfm.write_schema(con, images)
    cams = con.execute("SELECT camera_id, model, width, height, params, prior_focal_length FROM cameras").fetchall()
    assert len(cams) == 1 and cams[0][:4] == (1, 0, 40, 30) and cams[0][5] == 0
    assert np.frombuffer(cams[0][4], np.float64).tolist() == [48.0, 20.0, 15.0]
    rows = con.execute("SELECT * FROM images ORDER BY image_id").fetchall()
    assert [r[:3] for r in rows] == [(i + 1, n, 1) for i, n in enumerate(images.names)]
    assert all(v is None for r in rows for v in r[3:])
    assert con.execute("SELECT COUNT(*) FROM descriptors").fetchone()[0] == 0
    con.close()


def _exif(tag):
    e = Image.Exif()
    e.get_ifd(sfm.EXIF_IFD)[tag] = 4.5 if tag == 0x920A else 28
    return e


@pytest.mark.parametrize("case", ["subdir", "not_image", "size", "focal", "focal35", "empty", "frame", "single_camera"])
def test_refusals_before_any_library_call(tmp_path, no_library, case):
    img, out = tmp_path / "images", tmp_path / "out" / "sfm"
    num = 4
    if case == "focal":
        _frames(str(img), [(40, 30)] * num, fmt="jpg", exif=_exif(0x920A))
    elif case == "focal35":
        _frames(str(img), [(40, 30)] * num, fmt="jpg", exif=_exif(0xA405))
    elif case == "size":
        _frames(str(img), [(40, 30)] * (num - 1) + [(40, 31)])
    elif case == "empty":
        os.makedirs(img)
    else:
        _frames(str(img), [(40, 30)] * num)
    if case == "subdir":
        os.makedirs(img / "sub")
    if case == "not_image":
        (img / "notes.txt").write_text("not an image")
    tracks = _tracks(num)
    if case == "frame":
        tracks[7]["frame_ids"][-1] = num
    expect = {"subdir": "sub", "not_image": "notes.txt", "size": "00003.png", "focal": "FocalLength",
              "focal35": "FocalLengthIn35mmFilm", "empty": "no images", "frame": "trajectory 7",
              "single_camera": "single_camera"}[case]
    with pytest.raises(ValueError, match=expect):
        sfm.main_global_sfm(str(out), str(img), tracks, single_camera=case != "single_camera")
    assert not out.exists()


@pytest.mark.parametrize("flags", [["--sfm_type", "incremental_colmap"], ["--sfm_type", "global_glomap"],
                                   ["--single_camera", "0"], ["--skip_exists"]])
def test_cli_refuses_unsupported_flags(tmp_path, no_library, flags, capsys):
    assert sfm.main(["--image_dir", str(tmp_path), "--output_dir", str(tmp_path / "o")] + flags) == 2
    assert not (tmp_path / "o").exists()
    assert "not supported" in capsys.readouterr().err


@pytest.mark.parametrize("static", [False, True])
def test_cli_flags(tmp_path, monkeypatch, static):
    seen = {}

    def fake(sfm_dir, image_dir, traj_dir, **kw):
        seen.update(sfm_dir=sfm_dir, image_dir=image_dir, traj_dir=traj_dir, **kw)
        raise ValueError("stop")
    monkeypatch.setattr(sfm, "main_global_sfm", fake)
    o = str(tmp_path / "o")
    argv = ["--image_dir", "I", "--output_dir", o, "--skip_geometric_verification", "--min_num_matches", "30", "--quiet"]
    assert sfm.main(argv + (["--assume_static"] if static else [])) == 2
    assert seen["traj_dir"] == os.path.join(o, "trajectories" if static else "trajectories_labeled")
    assert seen["sfm_dir"] == os.path.join(o, "sfm") and seen["image_dir"] == "I"
    assert seen["remove_dynamic"] is (not static) and seen["skip_geometric_verification"] is True
    assert seen["min_num_matches"] == 30
    assert seen["convert_path"] == os.path.join(o, "colmap_outputs_converted")
    assert sfm.main(["--image_dir", "I", "--output_dir", o, "--traj_dir", "T", "--quiet"]) == 2
    assert seen["traj_dir"] == "T"
