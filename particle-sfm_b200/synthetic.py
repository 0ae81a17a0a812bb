"""Seeded synthetic workloads of the shapes named in BASELINE.json / SURVEY.md §8(d).

No dataset ships with the repo (no network): flows, trajectories and bundle-adjustment
problems are generated from geometry.  Used by tests/, bench.py and __graft_entry__.
"""
import numpy as np

from ._abi import BAProblem


# ----------------------------------------------------------------------------- rotations

def qvec_to_rotmat(q):
    """COLMAP convention, q = (w, x, y, z), vectorised over leading dims."""
    q = np.asarray(q, dtype=np.float64)
    w, x, y, z = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    R = np.empty(q.shape[:-1] + (3, 3))
    R[..., 0, 0] = 1 - 2 * (y * y + z * z)
    R[..., 0, 1] = 2 * (x * y - w * z)
    R[..., 0, 2] = 2 * (x * z + w * y)
    R[..., 1, 0] = 2 * (x * y + w * z)
    R[..., 1, 1] = 1 - 2 * (x * x + z * z)
    R[..., 1, 2] = 2 * (y * z - w * x)
    R[..., 2, 0] = 2 * (x * z - w * y)
    R[..., 2, 1] = 2 * (y * z + w * x)
    R[..., 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def rotmat_to_qvec(R):
    R = np.asarray(R, dtype=np.float64)
    flat = R.reshape(-1, 3, 3)
    out = np.empty((flat.shape[0], 4))
    for i, m in enumerate(flat):
        K = np.array([
            [m[0, 0] - m[1, 1] - m[2, 2], 0, 0, 0],
            [m[1, 0] + m[0, 1], m[1, 1] - m[0, 0] - m[2, 2], 0, 0],
            [m[2, 0] + m[0, 2], m[2, 1] + m[1, 2], m[2, 2] - m[0, 0] - m[1, 1], 0],
            [m[2, 1] - m[1, 2], m[0, 2] - m[2, 0], m[1, 0] - m[0, 1], m[0, 0] + m[1, 1] + m[2, 2]]]) / 3.0
        vals, vecs = np.linalg.eigh(K)
        q = vecs[[3, 0, 1, 2], np.argmax(vals)]
        if q[0] < 0:
            q = -q
        out[i] = q
    return out.reshape(R.shape[:-2] + (4,))


def axis_angle_to_rotmat(v):
    v = np.asarray(v, dtype=np.float64)
    th = np.linalg.norm(v, axis=-1, keepdims=True)
    k = np.divide(v, th, out=np.zeros_like(v), where=th > 0)
    K = np.zeros(v.shape[:-1] + (3, 3))
    K[..., 0, 1], K[..., 0, 2] = -k[..., 2], k[..., 1]
    K[..., 1, 0], K[..., 1, 2] = k[..., 2], -k[..., 0]
    K[..., 2, 0], K[..., 2, 1] = -k[..., 1], k[..., 0]
    s, c = np.sin(th)[..., None], np.cos(th)[..., None]
    return np.eye(3) + s * K + (1 - c) * (K @ K)


# ----------------------------------------------------------------------------- HP2

def make_ba_problem(num_images, num_points, track_len=12, seed=0, noise_px=0.5, focal=900.0,
                    cx=512.0, cy=218.0, center_noise=0.02, rot_noise_deg=0.5, point_noise=0.05,
                    track_len_range=None, dynamic_fraction=0.0, shuffle=True):
    """Global-BA stand-in (SURVEY.md §8d, config 5 generator): cameras on a 2-turn helix
    looking at the scene centroid, points uniform in a box in front of every camera, each
    point seen in a contiguous window of `track_len` frames (or U{lo..hi} when
    `track_len_range`), SIMPLE_PINHOLE shared by all images, observations = projection +
    N(0, noise_px^2) rounded to f32 (keypoints are stored f32, colmap_utils/database.py:185).
    Start = truth perturbed; gauge as the reference fixes it (sfm/global_mapper.cc:431-435):
    image 0 pose constant, image 1 tvec[0] constant.
    Returns (BAProblem, truth dict)."""
    rng = np.random.default_rng(seed)
    F, P = int(num_images), int(num_points)
    ang = np.linspace(0.0, 4.0 * np.pi, F)
    centres = np.stack([8.0 * np.cos(ang), 8.0 * np.sin(ang), np.linspace(-2.0, 2.0, F)], -1)
    zax = -centres / np.linalg.norm(centres, axis=1, keepdims=True)
    up = np.array([0.0, 0.0, 1.0])
    xax = np.cross(up, zax)
    xax /= np.linalg.norm(xax, axis=1, keepdims=True)
    yax = np.cross(zax, xax)
    R_true = np.stack([xax, yax, zax], 1)                       # world -> camera
    t_true = -np.einsum("fij,fj->fi", R_true, centres)
    q_true = rotmat_to_qvec(R_true)
    X_true = rng.uniform(-2.5, 2.5, size=(P, 3))

    if track_len_range is None:
        lens = np.full(P, min(int(track_len), F), dtype=np.int64)
    else:
        lo, hi = track_len_range
        lens = rng.integers(lo, min(hi, F) + 1, size=P)
    starts = (rng.random(P) * (F - lens + 1)).astype(np.int64)
    M = int(lens.sum())
    obs_point = np.repeat(np.arange(P, dtype=np.int64), lens)
    first = np.cumsum(lens) - lens
    obs_image = np.arange(M, dtype=np.int64) - np.repeat(first, lens) + np.repeat(starts, lens)
    if dynamic_fraction > 0:          # observations flagged dynamic are dropped before BA
        keep = rng.random(M) >= dynamic_fraction
        obs_point, obs_image = obs_point[keep], obs_image[keep]
        M = obs_point.shape[0]
    Xc = np.einsum("mij,mj->mi", R_true[obs_image], X_true[obs_point]) + t_true[obs_image]
    uv = Xc[:, :2] / Xc[:, 2:3]
    xy = focal * uv + np.array([cx, cy])
    xy = (xy + rng.normal(0.0, noise_px, size=xy.shape)).astype(np.float32).astype(np.float64)
    if shuffle:                        # the reference adds residuals image by image, not by point
        perm = rng.permutation(M)
        obs_point, obs_image, xy = obs_point[perm], obs_image[perm], xy[perm]

    # perturbed start
    c0 = centres + rng.normal(0.0, center_noise, size=centres.shape)
    dR = axis_angle_to_rotmat(rng.normal(size=(F, 3)) * np.deg2rad(rot_noise_deg) / np.sqrt(3.0))
    R0 = np.einsum("fij,fjk->fik", dR, R_true)
    R0[0], c0[0] = R_true[0], centres[0]
    q0 = rotmat_to_qvec(R0)
    t0 = -np.einsum("fij,fj->fi", R0, c0)
    X0 = X_true + rng.normal(0.0, point_noise, size=X_true.shape)
    pose_constant = np.zeros(F, np.uint8)
    pose_constant[0] = 1
    tmask = np.zeros(F, np.uint8)
    if F > 1:
        tmask[1] = 1
    prob = BAProblem(q0, t0, X0, np.array([[focal, cx, cy]]), obs_image.astype(np.int32),
                     obs_point.astype(np.int32), xy, np.zeros(F, np.int32), pose_constant, tmask,
                     np.zeros(1, np.uint8))
    truth = dict(qvec=q_true, tvec=t_true, xyz=X_true, centres=centres)
    return prob, truth


def camera_centres(qvec, tvec):
    """Image::ProjectionCenter() = -R(q)^T t."""
    R = qvec_to_rotmat(qvec)
    return -np.einsum("fji,fj->fi", R, np.asarray(tvec))


def umeyama_ate(est_centres, gt_centres):
    """ATE as evaluation_evo/eval_sintel.py:57-107 computes it through evo
    (align=True, correct_scale=True): Sim(3) Umeyama alignment of the estimated camera
    centres to ground truth, RMSE of the translation residuals."""
    x, y = np.asarray(est_centres, float), np.asarray(gt_centres, float)
    mx, my = x.mean(0), y.mean(0)
    xc, yc = x - mx, y - my
    cov = yc.T @ xc / x.shape[0]
    U, D, Vt = np.linalg.svd(cov)
    S = np.eye(3)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        S[2, 2] = -1
    R = U @ S @ Vt
    var_x = (xc ** 2).sum() / x.shape[0]
    s = np.trace(np.diag(D) @ S) / var_x
    t = my - s * R @ mx
    err = y - (s * (R @ x.T).T + t)
    return float(np.sqrt((err ** 2).sum(1).mean()))


# ----------------------------------------------------------------------------- a rigid video with exact flows

ROOM_HALF = np.array([4.0, 2.5, 4.0])          # the box room's half extents (x, y down, z)


def _room_camera(t, n_frames, seed_shift):
    """World-to-camera rotation R and centre C of frame t of the room sequence: a smooth path near the room's
    middle, turning left and right."""
    u = t / max(1, n_frames - 1)
    a, b = seed_shift
    c = np.array([-0.6 + 1.2 * u + 0.2 * a, 0.2 * np.sin(2 * np.pi * u + b), 0.4 * np.sin(np.pi * u) - 0.2])
    yaw, pitch = 0.15 * np.sin(np.pi * u + a) - 0.05, 0.04 * np.sin(2 * np.pi * u)
    cy, sy, cp, sp = np.cos(yaw), np.sin(yaw), np.cos(pitch), np.sin(pitch)
    ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    rx = np.array([[1, 0, 0], [0, cp, -sp], [0, sp, cp]])
    return (ry @ rx).T, c


def _room_points(R, C, h, w, camera):
    """The wall point seen at every pixel (i, j) (image point (j + 0.5, i + 0.5), COLMAP's pixel centre) from a
    camera inside the room: [h][w][3] world coordinates.  From inside a convex room every ray meets one wall."""
    f, cx, cy = camera
    jj, ii = np.meshgrid(np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64))
    d = np.stack([(jj + 0.5 - cx) / f, (ii + 0.5 - cy) / f, np.ones_like(jj)], -1) @ R       # rays in the world
    with np.errstate(divide="ignore"):
        hit = np.where(d > 0, (ROOM_HALF - C) / d, np.where(d < 0, (-ROOM_HALF - C) / d, np.inf))
    return C + hit.min(-1)[..., None] * d


def _room_texture(P, rng):
    """uint8 RGB of wall points: a few sinusoids of the 3D point per channel."""
    k = rng.uniform(-1, 1, (3, 4, 3)) * np.array([3.0, 7.0, 13.0, 23.0])[None, :, None]
    ph = rng.uniform(0, 2 * np.pi, (3, 4))
    amp = np.array([50.0, 35.0, 22.0, 12.0])
    out = np.empty(P.shape[:-1] + (3,))
    for c in range(3):
        out[..., c] = 128 + sum(amp[m] * np.sin(P @ k[c, m] + ph[c, m]) for m in range(4))
    return np.clip(np.rint(out), 0, 255).astype(np.uint8)


def _room_flow(P, R, C, camera):
    """Flow of the pixels whose world points are P [h][w][3] into the camera (R, C): the projection's pixel position
    minus the pixel's own; a point behind that camera gets a flow far outside the frame."""
    f, cx, cy = camera
    h, w = P.shape[:2]
    X = (P - C) @ R.T
    z = X[..., 2]
    front = z > 1e-9
    zs = np.where(front, z, 1.0)
    jj, ii = np.meshgrid(np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64))
    flow = np.stack([f * X[..., 0] / zs + cx - 0.5 - jj, f * X[..., 1] / zs + cy - 0.5 - ii], -1)
    flow[~front] = 1e6
    return flow.astype(np.float32)


def make_room_sequence(n_frames, h, w, seed=0):
    """A rigid video with exact flows: a camera (SIMPLE_PINHOLE, f = 1.2 max(w, h), principal point at the centre,
    what the SfM importer assumes) moves along a smooth path inside a convex box room, so no pixel is ever occluded;
    the walls are textured procedurally from the 3D point.  Returns (frames [n][h][w][3] uint8, flows {(t, stride):
    (forward, backward)} for strides 1 and 2, [h][w][2] float32 computed in closed form from every pixel's wall point
    and the two poses, qvec [n][4], tvec [n][3] (world to camera, COLMAP's convention))."""
    rng = np.random.default_rng(seed)
    camera = (1.2 * max(w, h), w / 2.0, h / 2.0)
    shift = rng.uniform(-1, 1, 2) * [0.5, np.pi]
    poses = [_room_camera(t, n_frames, shift) for t in range(n_frames)]
    tex = np.random.default_rng(rng.integers(1 << 31))
    frames, flows = [], {}
    pts = [_room_points(R, C, h, w, camera) for R, C in poses]
    tex_state = tex.bit_generator.state
    for P in pts:
        tex.bit_generator.state = tex_state                # the same texture on every frame
        frames.append(_room_texture(P, tex))
    for t in range(n_frames):
        for s in (1, 2):
            if t + s < n_frames:
                flows[(t, s)] = (_room_flow(pts[t], *poses[t + s], camera), _room_flow(pts[t + s], *poses[t], camera))
    qvec = np.array([rotmat_to_qvec(R) for R, _ in poses])
    tvec = np.array([-R @ C for R, C in poses])
    return np.stack(frames), flows, qvec, tvec


# ----------------------------------------------------------------------------- HP1

def bilinear_zeros(img, xy):
    """Bilinear sample of img [H,W,C] at xy [N,2] (x=col, y=row), zeros outside — the
    semantics of torch grid_sample(align_corners=True, padding_mode='zeros') that
    point_trajectory/trajectory.py:25-37 uses (here in float64; the bit-faithful float32
    version lives in tracker.py)."""
    img = np.asarray(img)
    H, W = img.shape[:2]
    x, y = xy[:, 0], xy[:, 1]
    x0, y0 = np.floor(x).astype(np.int64), np.floor(y).astype(np.int64)
    fx, fy = x - x0, y - y0
    out = np.zeros((xy.shape[0],) + img.shape[2:], dtype=np.float64)
    for dy, wy in ((0, 1 - fy), (1, fy)):
        for dx, wx in ((0, 1 - fx), (1, fx)):
            xi, yi = x0 + dx, y0 + dy
            ok = (xi >= 0) & (xi < W) & (yi >= 0) & (yi < H)
            v = img[np.clip(yi, 0, H - 1), np.clip(xi, 0, W - 1)].astype(np.float64)
            wgt = (wx * wy * ok)
            out += v * (wgt[:, None] if v.ndim == 2 else wgt)
    return out


def smooth_flow(height, width, rng, amplitude=6.0, waves=8):
    """Sum of `waves` low-frequency sinusoids, |flow| <= amplitude px (SURVEY.md §8d cfg 2)."""
    yy, xx = np.meshgrid(np.arange(height, dtype=np.float64), np.arange(width, dtype=np.float64),
                         indexing="ij")
    flow = np.zeros((height, width, 2))
    for _ in range(waves):
        kx, ky = rng.uniform(-3, 3, 2) * 2 * np.pi / np.array([width, height])
        ph = rng.uniform(0, 2 * np.pi, 2)
        a = rng.uniform(-1, 1, 2) * amplitude / waves
        flow[..., 0] += a[0] * np.sin(kx * xx + ky * yy + ph[0])
        flow[..., 1] += a[1] * np.sin(kx * xx + ky * yy + ph[1])
    return flow


def make_flow_triplet(height, width, seed=0, amplitude=6.0, noise=0.1):
    """flow01, flow12, flow02 (f32 [H,W,2]) with flow02 = flow01 + flow12∘(x+flow01) + noise,
    and an occlusion map for the stride-2 pair (bool [H,W], ~8% set)."""
    rng = np.random.default_rng(seed)
    f01 = smooth_flow(height, width, rng, amplitude)
    f12 = smooth_flow(height, width, rng, amplitude)
    yy, xx = np.meshgrid(np.arange(height, dtype=np.float64), np.arange(width, dtype=np.float64),
                         indexing="ij")
    p1 = np.stack([xx + f01[..., 0], yy + f01[..., 1]], -1).reshape(-1, 2)
    f12_at = bilinear_zeros(f12, p1).reshape(height, width, 2)
    f02 = f01 + f12_at + rng.normal(0, noise, size=f01.shape)
    f01n = f01 + rng.normal(0, noise, size=f01.shape)
    f12n = f12 + rng.normal(0, noise, size=f12.shape)
    occ02 = smooth_flow(height, width, rng, 1.0, 4)[..., 0] > 0.45
    return f01n.astype(np.float32), f12n.astype(np.float32), f02.astype(np.float32), occ02


def make_flow_sequence(n_frames, height, width, seed=0, amplitude=3.0, waves=4):
    """The four flow lists main_connect_point_trajectories takes for n_frames images, as
    tests/golden/make_tracker_golden.py builds them at any size: smooth forward flows fw [n-1],
    crude backward flows fb, two-step flows f2 [n-2] = fw[i] composed with fw[i+1] plus noise, their
    backward flows b2, and a block of extra motion moving across fw (not in fb) that the flow check
    marks occluded, so that particles die and new ones are seeded.  f32 [H, W, 2] each."""
    h, w = height, width
    rng = np.random.default_rng(seed)
    fw = [smooth_flow(h, w, rng, amplitude, waves).astype(np.float32) for _ in range(n_frames - 1)]
    yy, xx = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")

    def compose(a, b):   # a then b
        p = np.stack([xx + a[..., 0], yy + a[..., 1]], -1).reshape(-1, 2)
        return (a + bilinear_zeros(b, p).reshape(h, w, 2)).astype(np.float32)

    def backward(a):     # crude inverse: -a sampled at x - a
        p = np.stack([xx - a[..., 0], yy - a[..., 1]], -1).reshape(-1, 2)
        return (-bilinear_zeros(a, p).reshape(h, w, 2)).astype(np.float32)
    fb = [backward(f) for f in fw]
    f2 = [compose(fw[i], fw[i + 1]) + rng.normal(0, 0.05, (h, w, 2)).astype(np.float32) for i in range(n_frames - 2)]
    b2 = [backward(f) for f in f2]
    r0, r1 = (10 * h) // 36, (18 * h) // 36                  # the golden's rows 10:18 of 36
    c0, dc = (8 * w) // 52, max(1, (4 * w) // 52)            # its columns 8+4i : 16+4i of 52
    for i, f in enumerate(fw):
        f[r0:r1, c0 + dc * i:2 * c0 + dc * i] += 6.0
    return fw, fb, f2, b2


def make_traj_inputs(num, height, width, seed=0, amplitude=6.0, upper_flow=20.0):
    """The argument tuple IncrementalTrajectorySet.optimize_buffer hands to
    particlesfm.optimize_location (point_trajectory/trajectory.py:161-186) for `num`
    trajectories: uv12 [N,4], ref1 [N,2], ref2 [N,2], scale [N,1], flow12 [H,W,2] f32."""
    f01, f12, f02, occ02 = make_flow_triplet(height, width, seed, amplitude)
    rng = np.random.default_rng(seed + 1000003)
    x0 = np.stack([rng.uniform(8, width - 9, num), rng.uniform(8, height - 9, num)], -1)
    fl01 = bilinear_zeros(f01, x0)
    x1 = x0 + fl01
    x2 = x1 + bilinear_zeros(f12, x1)
    fl02 = bilinear_zeros(f02, x0)
    occ = bilinear_zeros(occ02.astype(np.float64)[..., None], x0)
    scale = (1.0 - occ) * (np.linalg.norm(fl02, axis=-1, keepdims=True) < upper_flow)
    # torch grid_sample returns float32; the reference then mixes into float64 arrays
    fl01 = fl01.astype(np.float32).astype(np.float64)
    fl02 = fl02.astype(np.float32).astype(np.float64)
    scale = scale.astype(np.float32).astype(np.float64)
    uv12 = np.concatenate([x1, x2], -1)
    return uv12, x0 + fl01, x0 + fl02, scale, f12


def make_track_arrays(num_trajs, num_frames, num_obs, seed=0, min_len=3, width=1024, height=436):
    """A seeded tracker.TrackArrays shaped like the tracker's output, with exactly `num_obs` observations:
    contiguous frame windows, geometric lengths clipped to [min_len, num_frames], then lengthened or shortened one
    observation at a time on random trajectories until the total matches."""
    from .tracker import TrackArrays
    if not min_len * num_trajs <= num_obs <= num_frames * num_trajs:
        raise ValueError("num_obs is out of reach of num_trajs trajectories of min_len .. num_frames observations")
    rng = np.random.default_rng(seed)
    lens = np.clip(rng.geometric(num_trajs / num_obs, num_trajs), min_len, num_frames).astype(np.int64)
    diff = num_obs - int(lens.sum())
    while diff:
        step = 1 if diff > 0 else -1
        cand = np.nonzero(lens < num_frames if step > 0 else lens > min_len)[0]
        pick = rng.choice(cand, min(abs(diff), cand.shape[0]), replace=False)
        lens[pick] += step
        diff -= step * pick.shape[0]
    start = (rng.random(num_trajs) * (num_frames - lens + 1)).astype(np.int64)
    ptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    frames = (np.arange(num_obs) - np.repeat(ptr[:-1], lens) + np.repeat(start, lens)).astype(np.int32)
    xy = rng.random((num_obs, 2)) * np.array([width - 1, height - 1], np.float64)
    return TrackArrays(np.arange(num_trajs, dtype=np.int64), ptr, frames, xy)


def make_two_view_scene(num_trajs, num_frames, num_obs, seed=0, focal=500.0, width=1024, height=436, step=0.02,
                        path="line"):
    """Static points seen by a camera that moves `step` per frame along x with a slow yaw: a tracker.TrackArrays with
    make_track_arrays' counts whose locations are the points' exact projections, minus the 0.5 that
    import_keypoints_matches adds back.  Every point lies 2 .. 40 in front of the camera at its first frame, so that
    between adjacent frames it is 100 .. 2000 baselines away: it straddles CheckCheirality's max_depth.
    path="helix" (opt-in) moves the camera on a helix about the x axis instead (x = step f, y and z on a circle of
    radius 4 step at 0.6 rad per frame): the centres are not near-collinear, which the global position estimation
    needs to be well conditioned.  The default path="line" is unchanged.
    Returns (tracks, qvec [F][4], tvec [F][3] world-to-camera, camera (f, cx, cy))."""
    tracks = make_track_arrays(num_trajs, num_frames, num_obs, seed=seed, width=width, height=height)
    rng = np.random.default_rng(seed + 1)
    f = np.arange(num_frames, dtype=np.float64)
    R = axis_angle_to_rotmat(np.stack([0.001 * f, 0.004 * f, np.zeros_like(f)], axis=1))
    if path == "line":
        centres = np.stack([step * f, 0.1 * step * np.sin(f), np.zeros_like(f)], axis=1)
    elif path == "helix":
        centres = step * np.stack([f, 4.0 * np.sin(0.6 * f), 4.0 * (1.0 - np.cos(0.6 * f))], axis=1)
    else:
        raise ValueError("path must be line or helix")
    tvec = -np.einsum("fij,fj->fi", R, centres)
    cam = np.array([focal, width / 2.0, height / 2.0])
    first = tracks.frame_ids[tracks.ptr[:-1]]
    px = rng.random((num_trajs, 2)) * np.array([width, height])
    depth = 2.0 + 38.0 * rng.random(num_trajs)
    Xc = np.stack([(px[:, 0] - cam[1]) / focal * depth, (px[:, 1] - cam[2]) / focal * depth, depth], axis=1)
    Xw = np.einsum("nji,nj->ni", R[first], Xc - tvec[first])
    X = np.repeat(Xw, np.diff(tracks.ptr), axis=0)
    fr = tracks.frame_ids
    Xcam = np.einsum("nij,nj->ni", R[fr], X) + tvec[fr]
    tracks.xy = focal * Xcam[:, :2] / Xcam[:, 2:] + cam[1:] - 0.5
    return tracks, rotmat_to_qvec(R), tvec, cam


def corrupt_keypoints(keypoints, fraction, seed=0, shift_px=(20.0, 60.0), noise_px=0.0):
    """Observation outliers for triangulation fixtures: a copy of keypoints [K][2] where a seeded `fraction` of them is
    moved by shift_px[0] .. shift_px[1] pixels in a random direction, and every keypoint gets Gaussian noise of
    noise_px.  Returns (keypoints, corrupted index array)."""
    rng = np.random.default_rng(seed)
    out = np.array(keypoints, np.float64).reshape(-1, 2)
    out += noise_px * rng.standard_normal(out.shape)
    idx = np.nonzero(rng.random(out.shape[0]) < fraction)[0]
    ang = rng.random(idx.shape[0]) * 2.0 * np.pi
    r = shift_px[0] + (shift_px[1] - shift_px[0]) * rng.random(idx.shape[0])
    out[idx] += np.stack([r * np.cos(ang), r * np.sin(ang)], 1)
    return out.astype(np.asarray(keypoints).dtype), idx


def relative_essential(qvec, tvec, a, b):
    """E = [t]x R of the relative pose from image a to image b (world-to-camera poses)."""
    Ra, Rb = qvec_to_rotmat(qvec[a]), qvec_to_rotmat(qvec[b])
    Rr = Rb @ Ra.T
    t = tvec[b] - Rr @ tvec[a]
    tx = np.array([[0.0, -t[2], t[1]], [t[2], 0.0, -t[0]], [-t[1], t[0], 0.0]])
    return tx @ Rr


def two_view_inputs(rows, image_ids, qvec, tvec, camera):
    """The arguments of init_geometry.estimate_relative_poses for handoff.DatabaseRows of one SIMPLE_PINHOLE camera:
    images in image_id order, pairs in row order, config CALIBRATED with E from the poses (qvec / tvec indexed by the
    position of the image in `image_ids`, a list of database ids); F = H = I."""
    order = np.argsort(image_ids)
    index = {int(image_ids[k]): r for r, k in enumerate(order)}
    kp = dict(rows.keypoints)
    kps = [kp[int(image_ids[k])] for k in order]
    from .handoff import pair_id_to_image_ids
    R = len(rows.matches)
    pair_images = np.zeros((R, 2), np.int32)
    E = np.zeros((R, 3, 3))
    for p, (pid, _) in enumerate(rows.matches):
        a, b = (index[int(i)] for i in pair_id_to_image_ids(pid))
        pair_images[p] = a, b
        E[p] = relative_essential(qvec, tvec, order[a], order[b])
    counts = np.array([m.shape[0] for _, m in rows.matches], np.int64)
    eye = np.broadcast_to(np.eye(3), (R, 3, 3))
    return dict(keypoint_ptr=np.concatenate([[0], np.cumsum([k.shape[0] for k in kps])]).astype(np.int64),
                keypoints=np.concatenate(kps) if kps else np.zeros((0, 2), np.float32),
                image_camera=np.zeros(len(image_ids), np.int32), cameras=np.asarray(camera, np.float64).reshape(1, 3),
                pair_images=pair_images, config=np.full(R, 2, np.int32), E=E, F=eye, H=eye,
                inlier_ptr=np.concatenate([[0], np.cumsum(counts)]).astype(np.int64),
                inlier_matches=np.concatenate([m for _, m in rows.matches]) if R else np.zeros((0, 2), np.uint32))


# ----------------------------------------------------------------------------- view graphs for rotation averaging

def _quat_mul(a, b):
    w1, x1, y1, z1 = np.moveaxis(a, -1, 0)
    w2, x2, y2, z2 = np.moveaxis(b, -1, 0)
    return np.stack([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                     w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2], -1)


def _axis_angle_quat(v):
    th = np.linalg.norm(v, axis=-1, keepdims=True)
    k = np.divide(v, th, out=np.zeros_like(v), where=th > 0)
    return np.concatenate([np.cos(0.5 * th), k * np.sin(0.5 * th)], -1)


def make_view_graph(num_images, graph="complete", band=10, noise_deg=0.0, outlier_fraction=0.0, seed=0,
                    num_isolated=0, unposed_fraction=0.0, max_angle_deg=30.0, direction_noise_deg=0.0,
                    direction_outlier_fraction=0.0):
    """A seeded view graph for rotation averaging.  Ground truth: world-to-camera orientations within max_angle_deg of
    the identity.  graph: "complete", "banded" (pairs up to `band` frames apart, a video) or "two_components" (images
    split 2 : 1, the larger half first, each half complete).  The last num_isolated images get no pair.  Each pair's
    2_R_1 = R2 R1^-1 is perturbed by a rotation of N(0, noise_deg) degrees about a random axis; an outlier_fraction of
    the pairs get a uniformly random rotation instead; an unposed_fraction get has_pose = 0.  num_correspondences is
    100 + 10 * (max(0, band - |a - b|) // 5): few distinct values, so many ties on purpose.
    Camera centres and pair translation directions come from a second generator, so every other key of a seed is
    the same with or without them: centres uniform in [-10, 10]^3, each pair's unit tvec = R2 (c1 - c2) / |c1 - c2|
    (the world-to-camera relative translation of the true poses), each component perturbed by N(0, direction_noise_deg)
    degrees and renormalised; a direction_outlier_fraction of the pairs get a uniformly random direction instead.
    Returns dict(num_images, pair_images [R][2], qvec [R][4], num_correspondences [R], has_pose [R], truth [F][4],
    outlier [R] bool, centres [F][3], tvec [R][3], direction_outlier [R] bool)."""
    rng = np.random.default_rng(seed)
    F = num_images
    axis = rng.normal(size=(F, 3))
    axis /= np.linalg.norm(axis, axis=1, keepdims=True)
    truth = _axis_angle_quat(axis * np.deg2rad(max_angle_deg) * rng.random((F, 1)))
    active = F - num_isolated
    if graph == "complete":
        groups = [range(active)]
    elif graph == "banded":
        groups = None
    elif graph == "two_components":
        cut = (2 * active) // 3
        groups = [range(cut), range(cut, active)]
    else:
        raise ValueError("graph must be complete, banded or two_components")
    if groups is None:
        pairs = [(a, b) for a in range(active) for b in range(a + 1, min(active, a + band + 1))]
    else:
        pairs = [(a, b) for g in groups for a in g for b in g if a < b]
    pairs = np.array(pairs, np.int32).reshape(-1, 2)
    R = pairs.shape[0]
    inv1 = truth[pairs[:, 0]] * np.array([1.0, -1.0, -1.0, -1.0])
    rel = _quat_mul(truth[pairs[:, 1]], inv1)
    if noise_deg > 0:
        ax = rng.normal(size=(R, 3))
        ax /= np.linalg.norm(ax, axis=1, keepdims=True)
        rel = _quat_mul(_axis_angle_quat(ax * np.deg2rad(noise_deg) * rng.normal(size=(R, 1))), rel)
    outlier = rng.random(R) < outlier_fraction
    if outlier.any():
        q = rng.normal(size=(int(outlier.sum()), 4))
        rel[outlier] = q / np.linalg.norm(q, axis=1, keepdims=True)
    gap = np.abs(pairs[:, 1] - pairs[:, 0])
    num_corr = (100 + 10 * (np.maximum(0, band - gap) // 5)).astype(np.int32)
    has_pose = (rng.random(R) >= unposed_fraction).astype(np.uint8)
    rng2 = np.random.default_rng([seed, 2])
    centres = rng2.uniform(-10.0, 10.0, (F, 3))
    t = np.einsum("rij,rj->ri", qvec_to_rotmat(truth[pairs[:, 1]]), centres[pairs[:, 0]] - centres[pairs[:, 1]])
    t /= np.linalg.norm(t, axis=1, keepdims=True)
    if direction_noise_deg > 0:
        t = t + np.deg2rad(direction_noise_deg) * rng2.normal(size=(R, 3))
        t /= np.linalg.norm(t, axis=1, keepdims=True)
    direction_outlier = rng2.random(R) < direction_outlier_fraction
    if direction_outlier.any():
        d = rng2.normal(size=(int(direction_outlier.sum()), 3))
        t[direction_outlier] = d / np.linalg.norm(d, axis=1, keepdims=True)
    return dict(num_images=F, pair_images=pairs, qvec=rel, num_correspondences=num_corr, has_pose=has_pose,
                truth=truth, outlier=outlier, centres=centres, tvec=t, direction_outlier=direction_outlier)
