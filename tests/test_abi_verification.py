"""psfm_verify_two_view_geometries at the C ABI: argument errors are decided on the host before any launch, so they hold
on a machine without a GPU; everything else needs the device."""
import os

import numpy as np
import pytest

from oracle import verification_oracle as vo
from particlesfm_b200 import _abi, _lib, device_count, init_geometry, launch_count
from test_oracle_verification import pair_tables, two_views


def _tables():
    return pair_tables([two_views(20, 1)[:2], two_views(20, 2)[:2]])


def _bad(name):
    mt = _tables()
    if name == "image index":
        mt.pair_images = np.array([[0, 1], [2, 4]], np.int32)
    elif name == "camera index":
        mt.image_camera = np.array([0, 1, 0, 0], np.int32)
    elif name == "keypoint index":
        mt.matches = mt.matches.copy()
        mt.matches[0, 0] = 20
    elif name == "with itself":
        mt.pair_images = np.array([[0, 1], [2, 2]], np.int32)
    elif name == "listed twice":
        mt.pair_images = np.array([[0, 1], [1, 0]], np.int32)
    elif name == "camera size":
        mt.camera_size = np.array([[1024, 0]])
    return mt


@pytest.mark.parametrize("why", ["image index", "camera index", "keypoint index", "with itself", "listed twice",
                                 "camera size"])
def test_bad_arguments_are_invalid_before_any_launch(why):
    n0 = launch_count()
    with pytest.raises(_lib.PsfmError) as e:
        init_geometry.verify_two_view_geometries(**_bad(why).verification_inputs())
    assert "status %d" % _abi.PSFM_ERR_INVALID in str(e.value) and why in str(e.value)
    assert launch_count() == n0


def test_options_check_and_calibrated_pairs_are_refused_before_any_launch():
    n0 = launch_count()
    for o in (dict(max_error=0.0), dict(min_num_trials=5, max_num_trials=4), dict(watermark_border_size=2.0)):
        with pytest.raises(_lib.PsfmError) as e:
            init_geometry.verify_two_view_geometries(**_tables().verification_inputs(),
                                                     options=init_geometry.TwoViewVerificationOptions(**o))
        assert "status %d" % _abi.PSFM_ERR_INVALID in str(e.value) and "Check()" in str(e.value)
    args = _tables().verification_inputs()
    args["prior_focal_length"] = np.ones(1, bool)
    with pytest.raises(_lib.PsfmError) as e:
        init_geometry.verify_two_view_geometries(**args)
    assert "status %d" % _abi.PSFM_ERR_UNSUPPORTED in str(e.value) and "prior focal length" in str(e.value)
    assert launch_count() == n0


def test_no_pair_launches_nothing():
    mt = _tables()
    mt.pair_images, mt.match_ptr, mt.matches = np.zeros((0, 2), np.int32), np.zeros(1, np.int64), np.zeros((0, 2), np.uint32)
    n0 = launch_count()
    r = init_geometry.verify_two_view_geometries(**mt.verification_inputs())
    assert launch_count() == n0 and r.config.shape == (0,) and r.inlier_ptr.tolist() == [0]
    assert r.summary["num_launches"] == 0


def test_defaults_agree_across_header_python_oracle_and_recalled():
    o = _abi.VerificationOptions()
    _lib.lib().psfm_verification_default_options(o)
    py = init_geometry.TwoViewVerificationOptions(max_error=2.0).to_struct()
    for name, _ in _abi.VerificationOptions._fields_:
        assert getattr(o, name) == vo.DEFAULTS[name], name
        assert getattr(py, name) == (2.0 if name == "max_error" else vo.DEFAULTS[name]), name
    here = os.path.dirname(_lib.__file__)
    header = open(os.path.join(here, os.pardir, "include", "psfm_b200.h")).read()
    struct = header.split("} psfm_verification_options;")[0].rsplit("typedef struct {", 1)[1]
    for name, value in vo.DEFAULTS.items():
        line = next(ln for ln in struct.splitlines() if (" %s;" % name) in ln)
        assert float(line.split("/*")[1].split()[0]) == value, name
    src = open(os.path.join(here, "csrc", "verification_recalled.cuh")).read()
    for name, key in (("kCapNumSamples", "ransac_cap_num_samples"), ("kMaxNumLocalTrials", "max_num_local_trials"),
                      ("kSevenPointSamples", "seven_point_samples"), ("kEightPointSamples", "eight_point_samples"),
                      ("kHomographySamples", "homography_samples"), ("kTranslationSamples", "translation_samples"),
                      ("kMinF22", "min_f22")):
        assert ("%s = %r;" % (name, vo.RECALLED[key])) in src, name


@pytest.mark.skipif(device_count() > 0, reason="checks the refusal without a device")
def test_no_device_is_refused():
    with pytest.raises(_lib.PsfmError) as e:
        init_geometry.verify_two_view_geometries(**_tables().verification_inputs())
    assert "status %d" % _abi.PSFM_ERR_NO_DEVICE in str(e.value) and "no CUDA device" in str(e.value)
