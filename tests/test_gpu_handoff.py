"""The track-set -> matches hand-off on the GPU (handoff.traj_to_matches_device, csrc/handoff.cu psfm_matches_*):
the same TrajectoryMatches, array for array, as the reference's output (tests/golden/handoff_small.npz) and as the host
function handoff.traj_to_matches, whose sampling rule for long strided tracks test_handoff.py pins."""
import numpy as np
import pytest

from particlesfm_b200 import _lib, handoff, synthetic as syn, tracker
from test_handoff import GOLD, _tracks

LENGTHS = (1, 2, 19, 20, 21, 39, 40, 41, 47, 100)
STRIDES = (1, 2, 5)


def _equal(d, h):
    assert d.num_images == h.num_images and len(d.keypoints) == len(h.keypoints) == h.num_images
    for a, b in zip(d.keypoints, h.keypoints):
        assert a.dtype == b.dtype == np.float64 and a.shape == b.shape and np.array_equal(a, b)
    for name in ("pair_images", "pair_ptr", "matches"):
        a, b = getattr(d, name), getattr(h, name)
        assert a.dtype == b.dtype and a.shape == b.shape, name
        assert np.array_equal(a, b), name


def _seeded(seed, num_images=530, dynamic=0.2):
    """Every length of LENGTHS at every stride of STRIDES, twice, in random windows of frames 8 .. 509, ~20 % dynamic
    samples, two fully dynamic trajectories, keys in no particular order: frames 0 .. 7 and 510 .. 529 hold no sample."""
    rng = np.random.default_rng(seed)
    tracks = {}
    keys = rng.permutation(10 ** 6)[:200].tolist()
    specs = [(n, s) for n in LENGTHS for s in STRIDES] * 2 + [(5, 1), (30, 2)]
    for idx, (n, s) in enumerate(specs):
        start = int(rng.integers(8, 510 - (n - 1) * s))
        labels = (rng.random(n) < dynamic).astype(np.int64)
        if idx >= len(specs) - 2:
            labels[:] = 1
        tracks[keys[idx]] = {"locations": (rng.random((n, 2)) * 500).tolist(), "labels": labels.tolist(),
                             "frame_ids": (start + s * np.arange(n)).tolist()}
    return tracks, num_images


@pytest.mark.gpu
@pytest.mark.parametrize("tag,remove_dynamic", [("static", True), ("all", False)])
def test_device_equals_the_reference_golden(gpu, tag, remove_dynamic):
    g = np.load(GOLD)
    n = int(g["num_images"])
    m = handoff.traj_to_matches_device(_tracks(g), n, remove_dynamic=remove_dynamic)
    kp_ptr = g[f"{tag}_kp_ptr"]
    for i in range(n):
        assert np.array_equal(m.keypoints[i], g[f"{tag}_kp"][kp_ptr[i]:kp_ptr[i + 1]])
    assert np.array_equal(m.pair_images, g[f"{tag}_pairs"])
    assert np.array_equal(m.pair_ptr, g[f"{tag}_pair_ptr"])
    assert np.array_equal(m.matches, g[f"{tag}_matches"])
    _equal(m, handoff.traj_to_matches(_tracks(g), n, remove_dynamic=remove_dynamic))


@pytest.mark.gpu
@pytest.mark.parametrize("sample_k", [1, 2, 20])
@pytest.mark.parametrize("remove_dynamic", [True, False])
def test_device_equals_host_on_seeded_track_sets(gpu, sample_k, remove_dynamic):
    tracks, num_images = _seeded(sample_k * 10 + remove_dynamic)
    h = handoff.traj_to_matches(tracks, num_images, remove_dynamic=remove_dynamic, sample_k=sample_k)
    assert all(k.shape == (0, 2) for k in h.keypoints[:8] + h.keypoints[510:])
    assert h.matches.shape[0] > 0
    _equal(handoff.traj_to_matches_device(tracks, num_images, remove_dynamic=remove_dynamic, sample_k=sample_k), h)


@pytest.mark.gpu
def test_device_empty_and_all_dynamic_track_sets(gpu):
    launches = _lib.lib().psfm_launch_count()
    all_dynamic = {3: {"locations": [[1.0, 2.0], [3.0, 4.0]], "labels": [1, 1], "frame_ids": [0, 1]}}
    for tracks, n in (({}, 0), ({}, 4), (all_dynamic, 4)):
        _equal(handoff.traj_to_matches_device(tracks, n), handoff.traj_to_matches(tracks, n))
    assert _lib.lib().psfm_launch_count() == launches                  # nothing was launched


@pytest.mark.gpu
def test_device_single_sample_trajectories_are_keypoints(gpu):
    tracks = {k: {"locations": [[float(k), 1.0]], "labels": [0], "frame_ids": [k % 3]} for k in range(7)}
    d = handoff.traj_to_matches_device(tracks, 3)
    _equal(d, handoff.traj_to_matches(tracks, 3))
    assert d.matches.shape == (0, 2) and [k.shape[0] for k in d.keypoints] == [3, 2, 2]


@pytest.mark.gpu
def test_device_on_the_resident_tracker_output(gpu):
    fw, fb, f2, b2 = syn.make_flow_sequence(8, 64, 96, seed=4)
    arrays = tracker.main_connect_point_trajectories_device(fw, fb, f2, b2, 2, 1.0, 3)
    assert isinstance(arrays, tracker.TrackArrays) and arrays.ptr[-1] > 0
    for num_images in (8, 12):
        _equal(handoff.traj_to_matches_device(arrays, num_images), handoff.traj_to_matches(arrays, num_images))


@pytest.mark.gpu
def test_device_equals_host_on_a_million_observations(gpu):
    arrays = syn.make_track_arrays(25000, 60, 1_000_000, seed=2)
    h = handoff.traj_to_matches(arrays, 60)
    d = handoff.traj_to_matches_device(arrays, 60)
    assert h.matches.shape[0] > 10 ** 7
    _equal(d, h)
    names = ["%05d.png" % i for i in range(60)]
    image_ids = {name: 60 - i for i, name in enumerate(names)}
    a = handoff.import_keypoints_matches_arrays(names, image_ids, d, True)
    b = handoff.import_keypoints_matches_arrays(names, image_ids, h, True)
    assert [i for i, _ in a.matches] == [i for i, _ in b.matches]
    assert all(x.tobytes() == y.tobytes() for (_, x), (_, y) in zip(a.matches, b.matches))


@pytest.mark.gpu
@pytest.mark.parametrize("frame", [-1, 5, 2 ** 33])
def test_device_refuses_out_of_range_frames(gpu, frame):
    tracks = {0: {"locations": [[1.0, 2.0], [3.0, 4.0], [5.0, 6.0]], "labels": [0, 0, 0], "frame_ids": [0, frame, 2]}}
    with pytest.raises(_lib.PsfmError, match="outside"):
        handoff.traj_to_matches_device(tracks, 5)
    with pytest.raises(_lib.PsfmError, match="sample_k"):
        handoff.traj_to_matches_device({}, 5, sample_k=0)
