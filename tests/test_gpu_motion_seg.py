"""The trajectory labeller on the GPU (particlesfm_b200.motion_seg, csrc/motion_seg.cu) against the host restatement
oracle/motion_seg_oracle.py."""
import hashlib
import os

import numpy as np
import pytest

import oracle.motion_seg_oracle as O

pytestmark = pytest.mark.gpu

# the fused encoder against nn.Transformer on the CPU: fp32 with reordered sums, exp and rsqrt
FEAT_ATOL = 2e-4
# labels are compared where the oracle's logit is farther than this from 0
LOGIT_MARGIN = 1e-3


@pytest.fixture(autouse=True)
def no_tf32():
    import torch
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = old


def _device_csr(tracks):
    import torch
    ids, ptr, frames, xy = tracks.csr()
    return ids, torch.from_numpy(ptr).cuda(), torch.from_numpy(frames).cuda(), torch.from_numpy(xy).cuda()


@pytest.mark.parametrize("length,window,cap", [(12, 5, 100000), (12, 5, 40), (12, 20, 100000), (7, 3, 25)])
def test_sampler_equals_the_track_set(length, window, cap):
    from particlesfm_b200 import motion_seg
    tracks = O.seeded_track_set(300, length, 96, 160, seed=11)
    tracks.build_invert_indexes()
    ids, ptr, frames, xy = _device_csr(tracks)
    win = motion_seg.sample_windows(ptr, frames, xy, length, window, cap)
    loc, valid, rows = win.loc.cpu().numpy(), win.valid.cpu().numpy(), win.rows.cpu().numpy()
    for w, idx in enumerate(O.windows(length, window)):
        s = tracks.sample_inside_window(idx, 3, cap)
        a, b = win.bounds[w], win.bounds[w + 1]
        assert ids[rows[a:b]].tolist() == list(s["traj_ids"])
        assert np.array_equal(valid[a:b], s["masks"].astype(np.uint8))
        assert np.array_equal(loc[a:b, :, 0], s["locations"][0]) and np.array_equal(loc[a:b, :, 1], s["locations"][1])


@pytest.mark.parametrize("h,w", [(96, 160), (480, 854), (436, 1024), (1080, 1920)])
def test_depth_resize_is_cv2_bit_for_bit(h, w):
    import torch
    from particlesfm_b200 import motion_seg
    px = O.seeded_depth_pixels(2, h, w, seed=h)
    got = motion_seg.depth_resize(torch.from_numpy(px).cuda()).cpu().numpy()
    for i in range(2):
        assert np.array_equal(got[i], O.depth_map(px[i]))


def _rows(K, L, seed, raw=(96, 160)):
    rng = np.random.default_rng(seed)
    valid = (rng.uniform(size=(K, L)) > 0.3).astype(np.uint8)
    valid[:, :min(3, L)] = 1
    rng.shuffle(valid, axis=1)
    loc = np.stack([rng.uniform(0, raw[1], (K, L)), rng.uniform(0, raw[0], (K, L))], -1)
    loc[:, 0, 0] = raw[1]                       # x = 1.0 after normalising: the gather wraps to the next row
    loc[valid == 0] = 0
    return loc, valid


@pytest.mark.parametrize("K", [1, 2, 33, 100000])
@pytest.mark.parametrize("L", [3, 10, 17])
def test_fused_encoder_matches_nn_transformer(K, L):
    import torch
    from particlesfm_b200 import motion_seg
    if K == 100000 and L != 10:
        pytest.skip("the full-size window runs at the default length only")
    raw = (96, 160)
    sd = O.seeded_state_dict(3)
    sdf = {k: v.float() for k, v in sd.items() if not k.endswith("num_batches_tracked")}
    loc, valid = _rows(K, L, seed=K + L, raw=raw)
    depth = O.seeded_depth_pixels(L, 24, 40, seed=5)
    maps = np.stack([O.depth_map(p) for p in depth])
    win = motion_seg.Windows()
    win.L = L
    win.starts = torch.zeros(1, dtype=torch.int32, device="cuda")
    win.rows = torch.zeros(K, dtype=torch.int32, device="cuda")
    win.row_window = torch.zeros(K, dtype=torch.int32, device="cuda")
    win.loc = torch.from_numpy(loc).cuda()
    win.valid = torch.from_numpy(valid).cuda()
    packed = torch.from_numpy(motion_seg.pack_encoder(sdf)).cuda()
    got = motion_seg.encode(win, torch.from_numpy(maps).cuda(), raw, packed).cpu()
    nor = loc.copy()
    nor[..., 0] = nor[..., 0] / (raw[1] / 424.0) / 424
    nor[..., 1] = nor[..., 1] / (raw[0] / 240.0) / 240
    nor = np.clip(nor, 0, 1).astype(np.float32)
    ref = torch.empty(K, 16)
    model = O.transformer(sd)
    for a in range(0, K, 4096):
        b = min(K, a + 4096)
        _, proj, _ = O.features(sdf, maps, nor[a:b], valid[a:b])
        ref[a:b] = O.encode(model, proj, valid[a:b])
    err = (got - ref).abs().max().item()
    print("K=%d L=%d: max |fused - nn.Transformer| = %.3g" % (K, L, err))
    assert err <= FEAT_ATOL


def _write_inputs(root, n, h, w, tracks, sd):
    import cv2
    import torch
    img, dep, trj = (os.path.join(root, d) for d in ("images", "midas_depth", "trajectories"))
    for d in (img, dep, trj):
        os.makedirs(d)
    frames = O.seeded_frames(n, h, w, seed=9)
    px = O.seeded_depth_pixels(n, h, w, seed=8)
    for i in range(n):
        cv2.imwrite(os.path.join(img, "%05d.png" % i), frames[i][:, :, ::-1])
        cv2.imwrite(os.path.join(dep, "%05d.png" % i), px[i])
    np.save(os.path.join(trj, "track.npy"), tracks)
    torch.save({"model_state_dict": sd}, os.path.join(root, "ckpt.pth"))
    return img, dep, trj, frames, px


@pytest.mark.parametrize("n,window,cap", [(12, 5, 100000), (12, 5, 30), (6, 10, 100000)])
def test_stage_equals_the_oracle(tmp_path, n, window, cap):
    import cv2
    from particlesfm_b200 import motion_seg
    h, w = 96, 160                                  # frames and depth maps are up-scaled to 240 x 424
    sd = O.seeded_state_dict(4)
    tracks = O.seeded_track_set(200, n, h, w, seed=n + window)
    img, dep, trj, frames, px = _write_inputs(str(tmp_path), n, h, w, tracks, sd)
    out_dir = str(tmp_path / "labeled")
    assert motion_seg.main(["--image_dir", img, "--depth_dir", dep, "--traj_dir", trj, "--output_traj_dir", out_dir,
                            "--model", str(tmp_path / "ckpt.pth"), "--window_size", str(window),
                            "--traj_max_num", str(cap)]) == 0
    got = np.load(os.path.join(out_dir, "track.npy"), allow_pickle=True).item()
    ref, wins, video = O.label(
        (h, w), px, O.seeded_track_set(200, n, h, w, seed=n + window), sd, window, cap, frames)
    assert list(got.keys()) == list(ref.keys())
    assert all(type(a) is type(b) for a, b in zip(got.keys(), ref.keys()))
    for k in ref:
        assert np.array_equal(got[k]["frame_ids"], ref[k]["frame_ids"])
        assert got[k]["frame_ids"].dtype == np.int64 and got[k]["labels"].dtype == bool
        assert np.array_equal(got[k]["locations"], ref[k]["locations"])
    g = np.concatenate([got[k]["labels"] for k in ref])
    r = np.concatenate([ref[k]["labels"] for k in ref])
    decided = np.abs(O.deciding_logits(ref, wins, window, n)) > LOGIT_MARGIN
    print("label flips: %d of %d observations, %d observations decided within %g of 0"
          % (int(np.sum(g != r)), g.size, int(np.sum(~decided)), LOGIT_MARGIN))
    assert np.array_equal(g[decided], r[decided])
    cap_ = cv2.VideoCapture(os.path.join(out_dir, "motion_seg.mp4"))
    count = 0
    while cap_.read()[0]:
        count += 1
    assert count == len(video) == sum(len(i) for i in O.windows(n, window))
    # the frames before encoding, through label_trajectories' sink, equal the oracle's cv2 drawing byte for byte
    import torch
    hashes = []

    def sink(meta, out):
        hashes.extend(hashlib.sha256(np.ascontiguousarray(f).tobytes()).hexdigest() for f in out.cpu().numpy())
    _, raw_hw, resized = motion_seg.frame_list(img)
    motion_seg.label_trajectories(motion_seg.read_tracks(trj), torch.from_numpy(px).cuda(), raw_hw,
                                  motion_seg.load_weights(str(tmp_path / "ckpt.pth")), window, cap, sink,
                                  torch.from_numpy(resized).cuda())
    if np.array_equal(g, r):
        assert hashes == [hashlib.sha256(np.ascontiguousarray(f).tobytes()).hexdigest() for f in video]


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "motion_seg_small.npz")
# OANet's convolutions at torch's defaults (cuDNN TF32, inputs rounded to 10-bit mantissas, 2^-11 relative) against
# the reference's float32 CPU logits, through 26 convolutions, each after an instance norm that rescales its input's
# spread to 1: a few per cent of the largest logit (2.0e-2 measured on the H100 at 700 W)
TF32_LOGIT_RTOL = 5e-2


def test_oanet_at_tf32_defaults_stays_near_the_reference():
    import torch
    from particlesfm_b200 import motion_seg
    g = np.load(GOLDEN)
    sd = {k: v.cuda() for k, v in motion_seg.check_state_dict({"model_state_dict": O.seeded_state_dict(4)},
                                                              "seeded").items()}
    torch.backends.cudnn.allow_tf32 = True
    worst = 0.0
    for f in [f for f in g.files if f.startswith("feat_")]:
        ref = g[f.replace("feat_", "logit_")]
        with torch.no_grad():
            got = motion_seg.oanet_logits(sd, torch.from_numpy(g[f]).cuda()).cpu().numpy()
        worst = max(worst, float(np.abs(got - ref).max() / max(np.abs(ref).max(), 1.0)))
    print("OANet at TF32 defaults: max |logit - reference| / max |logit| = %.3g" % worst)
    assert worst <= TF32_LOGIT_RTOL


def test_merge_equals_the_reference_loop():
    import torch
    from particlesfm_b200 import motion_seg
    n, window = 12, 5
    tracks = O.seeded_track_set(300, n, 96, 160, seed=21)
    ids, ptr, frames, xy = _device_csr(tracks)
    win = motion_seg.sample_windows(ptr, frames, xy, n, window, 40)
    pred = torch.from_numpy(np.random.default_rng(1).integers(0, 2, win.rows.shape[0]).astype(bool)).cuda()
    labels, first = motion_seg.merge(ptr, frames, win, pred)
    labels, first = labels.cpu().numpy(), first.cpu().numpy()
    rows, valid, p = win.rows.cpu().numpy(), win.valid.cpu().numpy(), pred.cpu().numpy()
    h_ptr, h_frames = ptr.cpu().numpy(), frames.cpu().numpy()
    want, order = {}, []                           # main_motion_segmentation's merge loop, restated
    for w, idx in enumerate(O.windows(n, window)):
        for r in range(win.bounds[w], win.bounds[w + 1]):
            t = int(rows[r])
            if t not in want:
                want[t] = {}
                order.append(t)
            for j, f in enumerate(idx):
                if valid[r, j] and f not in want[t]:
                    want[t][f] = int(p[r])
    assert [t for t in np.argsort(np.where(first >= 0, first, 1 << 30), kind="stable")[:len(order)]] == order
    for t in range(len(h_ptr) - 1):
        for j in range(h_ptr[t], h_ptr[t + 1]):
            assert labels[j] == want.get(t, {}).get(int(h_frames[j]), -1)


def test_drawn_frames_equal_cv2(tmp_path):
    import torch
    from particlesfm_b200 import motion_seg
    raw = (240, 424)
    L, K = 4, 40
    rng = np.random.default_rng(3)
    loc, valid = _rows(K, L, seed=4, raw=raw)
    # centres on and beyond every border
    loc[0, :, :] = [[0, 0], [423.9, 0], [0, 239.9], [424, 240]]
    loc[1, :, :] = [[1, 120], [422, 120], [200, 1], [200, 238]]
    valid[:2] = 1
    pred = rng.integers(0, 2, K).astype(bool)
    frames = O.seeded_frames(L, 240, 424, seed=6)
    draws = np.random.RandomState(0).randint(K, size=100).tolist()
    got = motion_seg.draw_window(torch.from_numpy(frames).cuda(), torch.from_numpy(loc).cuda(),
                                 torch.from_numpy(valid).cuda(), torch.from_numpy(pred).cuda(), raw, draws).cpu().numpy()
    import cv2
    colors = O.motion_seg_colors()
    for j in range(L):
        rows = [frames[j].copy() for _ in range(3)]
        for i in range(K):
            if valid[i, j]:
                c = (int(min(max(loc[i, j, 0] / 424, 0), 1) * 424), int(min(max(loc[i, j, 1] / 240, 0), 1) * 240))
                cv2.circle(rows[0], c, 1, colors[int(pred[i])], 2)
                cv2.circle(rows[1], c, 1, colors[0], 1)
        for i in draws:
            if valid[i, j]:
                c = (int(min(max(loc[i, j, 0] / 424, 0), 1) * 424), int(min(max(loc[i, j, 1] / 240, 0), 1) * 240))
                cv2.circle(rows[2], c, 3, colors[i % 6], 4)
        ref = np.concatenate([frames[j]] + rows, 0)
        assert np.array_equal(got[j], ref), j
