"""import_keypoints_matches_arrays: the COLMAP rows of the reference's import_keypoints_matches
(sfm/import_feature_matches.py:76-104) taken straight from a TrajectoryMatches, equal row for row to the list path
and byte-identical to the rows the reference left in its database (tests/golden/import_small.npz); and the device
hand-off refuses to run without a GPU."""
import numpy as np
import pytest

from particlesfm_b200 import _lib, handoff
from test_handoff import GOLD, _tracks
from test_import_matches import _inputs


def _same_rows(x, y):
    for a, b in ((x.keypoints, y.keypoints), (x.matches, y.matches), (x.two_view, y.two_view)):
        assert len(a) == len(b)
        for (ia, ra), (ib, rb) in zip(a, b):
            assert ia == ib and ra.dtype == rb.dtype and ra.shape == rb.shape and ra.tobytes() == rb.tobytes()
            assert ra.flags.c_contiguous


def _matches(remove_dynamic=True):
    g = np.load(GOLD)
    n = int(g["num_images"])
    return handoff.traj_to_matches(_tracks(g), n, remove_dynamic=remove_dynamic), ["%05d.png" % i for i in range(n)]


@pytest.mark.parametrize("skip", [False, True])
@pytest.mark.parametrize("remove_dynamic", [True, False])
@pytest.mark.parametrize("id_order", ["sorted", "reversed", "shuffled"])
def test_arrays_equal_the_list_path(skip, remove_dynamic, id_order):
    m, names = _matches(remove_dynamic)
    ids = list(range(1, len(names) + 1))
    order = list(names)
    if id_order == "reversed":
        ids = ids[::-1]
    elif id_order == "shuffled":
        rng = np.random.default_rng(5)
        ids = rng.permutation(ids).tolist()
        order = [names[k] for k in rng.permutation(len(names))]       # the dict's iteration order differs from the names
    image_ids = {name: ids[names.index(name)] for name in order}
    ref = handoff.import_keypoints_matches(image_ids, m.as_reference(names), skip_geometric_verification=skip)
    got = handoff.import_keypoints_matches_arrays(names, image_ids, m, skip_geometric_verification=skip)
    _same_rows(got, ref)


@pytest.mark.parametrize("skip", [False, True])
def test_arrays_equal_the_reference_database(skip):
    gi, data, image_ids = _inputs()
    g = np.load(GOLD)
    n = int(g["num_images"])
    names = ["%05d.png" % i for i in range(n)]
    m = handoff.traj_to_matches(_tracks(g), n)
    rows = handoff.import_keypoints_matches_arrays(names, image_ids, m, skip_geometric_verification=skip)
    _same_rows(rows, handoff.import_keypoints_matches(image_ids, data, skip_geometric_verification=skip))
    tag = "skip" if skip else "verify"
    gk = {gid: (r, c, blob) for gid, r, c, blob in gi[tag + "_keypoints"]}
    gm = {gid: (r, c, blob) for gid, r, c, blob in gi[tag + "_matches"]}
    gt = {x[0]: tuple(x[1:]) for x in gi[tag + "_two_view"]}
    assert len(rows.keypoints) == len(gk) and len(rows.matches) == len(gm) and len(rows.two_view) == len(gt)
    for iid, k in rows.keypoints:
        assert (k.shape[0], k.shape[1], k.tobytes()) == gk[iid]
    for pid, mm in rows.matches:
        assert mm.dtype == np.uint32 and (mm.shape[0], mm.shape[1], mm.tobytes()) == gm[pid]
    for pid, mm in rows.two_view:
        assert mm.tobytes() == gt[pid][2]


def test_arrays_of_an_empty_track_set():
    m = handoff.traj_to_matches({}, 3)
    names = ["a", "b", "c"]
    rows = handoff.import_keypoints_matches_arrays(names, {"c": 3, "a": 1, "b": 2}, m, True)
    assert [i for i, _ in rows.keypoints] == [3, 1, 2] and all(k.shape == (0, 2) and k.dtype == np.float32 for _, k in rows.keypoints)
    assert rows.matches == [] and rows.two_view == []


@pytest.mark.skipif(_lib.lib().psfm_device_count() > 0, reason="needs a machine WITHOUT a GPU")
def test_device_hand_off_has_no_cpu_fallback():
    g = np.load(GOLD)
    with pytest.raises(_lib.PsfmError, match="no CUDA device"):
        handoff.traj_to_matches_device(_tracks(g), int(g["num_images"]))
