"""TEST INFRASTRUCTURE (never imported by the product): numpy restatement of the relative-pose step that
gcolmap's DatabaseCache::Load runs per verified image pair (base/database_cache.cc:206-228):
TwoViewGeometry::EstimateRelativePose (estimators/two_view_geometry.cc:172-239) with PoseFromEssentialMatrix,
DecomposeEssentialMatrix, PoseFromHomographyMatrix, DecomposeHomographyMatrix, CheckCheirality,
TriangulatePoint, CalculateDepth, CalculateTriangulationAngles, RotationMatrixToQuaternion (Eigen's
Quaterniond(Matrix3d)) and Median of COLMAP bd84ad6 (not vendored).  Parity unpinned: pinned by the
known-answer tests of tests/test_oracle_two_view.py.

Two corners are defined here, as in csrc/two_view.cu:
* candidate order of an essential matrix.  Its SVD is not unique (sigma1 = sigma2 for an exact essential matrix,
  and u3, v3 have no common sign when sigma3 = 0), and only the order of the four candidates depends on it.  The
  order is fixed on the candidates themselves: t has its largest-magnitude component positive (ties to the lower
  index), R1 is the rotation of larger trace (equal traces keep the SVD's order).  It decides between candidates
  whose counts tie, nothing else.
* no homography candidate keeps a point (a pure rotation, whose single candidate has t = 0 and so max_depth = 0):
  the reference leaves R unset; here candidate 0 is taken, with tri_angle 0.
"""
import numpy as np

from .refine_oracle import triangulation_angle

CALIBRATED, UNCALIBRATED, PLANAR, PANORAMIC, PLANAR_OR_PANORAMIC = 2, 3, 4, 5, 6
ESTIMATED_CONFIGS = (CALIBRATED, UNCALIBRATED, PLANAR, PANORAMIC, PLANAR_OR_PANORAMIC)
EPS = np.finfo(np.float64).eps
W = np.array([[0.0, 1.0, 0.0], [-1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])


def calibration(cam):
    f, cx, cy = (float(v) for v in cam)
    return np.array([[f, 0.0, cx], [0.0, f, cy], [0.0, 0.0, 1.0]])


def image_to_world(cam, xy):
    """SIMPLE_PINHOLE ImageToWorld in fp64."""
    f, cx, cy = (float(v) for v in cam)
    xy = np.asarray(xy, np.float64).reshape(-1, 2)
    return np.stack([(xy[:, 0] - cx) / f, (xy[:, 1] - cy) / f], axis=1)


def canonical_t(t):
    """t with its largest-magnitude component positive (ties to the lower index)."""
    i = int(np.argmax(np.abs(t)))
    return -t if t[i] < 0 else t


def decompose_essential_matrix(E):
    """DecomposeEssentialMatrix, then the candidate order of the module docstring: [(R1, t), (R2, t), (R1, -t), (R2, -t)]."""
    U, _, V = np.linalg.svd(np.asarray(E, np.float64))       # V = svd.matrixV().transpose()
    if np.linalg.det(U) < 0:
        U = -U
    if np.linalg.det(V) < 0:
        V = -V
    R1, R2 = U @ W @ V, U @ W.T @ V
    t = canonical_t(U[:, 2] / np.linalg.norm(U[:, 2]))
    if np.trace(R2) > np.trace(R1):
        R1, R2 = R2, R1
    return [(R1, t), (R2, t), (R1, -t), (R2, -t)]


def _opposite_of_minor(S, row, col):
    c1, c2 = (1 if col == 0 else 0), (1 if col == 2 else 2)
    r1, r2 = (1 if row == 0 else 0), (1 if row == 2 else 2)
    return S[r1, c2] * S[r2, c1] - S[r1, c1] * S[r2, c2]


def decompose_homography_matrix(H, K1, K2):
    """DecomposeHomographyMatrix: [(R1, t1), (R1, -t1), (R2, t2), (R2, -t2)], or [(Hn, 0)] for a rotation."""
    Hn = np.linalg.inv(K2) @ np.asarray(H, np.float64) @ K1
    Hn = Hn / np.linalg.svd(Hn, compute_uv=False)[1]
    if np.linalg.det(Hn) < 0:
        Hn = -Hn
    S = Hn.T @ Hn - np.eye(3)
    if np.abs(S).max() < 1e-3:
        return [(Hn, np.zeros(3))]
    M00, M11, M22 = (_opposite_of_minor(S, i, i) for i in range(3))
    rt00, rt11, rt22 = np.sqrt(M00), np.sqrt(M11), np.sqrt(M22)
    e12, e02, e01 = (float(np.sign(_opposite_of_minor(S, a, b))) for a, b in ((1, 2), (0, 2), (0, 1)))
    idx = int(np.argmax(np.abs(np.diag(S))))
    if idx == 0:
        np1 = np.array([S[0, 0], S[0, 1] + rt22, S[0, 2] + e12 * rt11])
        np2 = np.array([S[0, 0], S[0, 1] - rt22, S[0, 2] - e12 * rt11])
    elif idx == 1:
        np1 = np.array([S[0, 1] + rt22, S[1, 1], S[1, 2] - e02 * rt00])
        np2 = np.array([S[0, 1] - rt22, S[1, 1], S[1, 2] + e02 * rt00])
    else:
        np1 = np.array([S[0, 2] + e01 * rt11, S[1, 2] + rt00, S[2, 2]])
        np2 = np.array([S[0, 2] - e01 * rt11, S[1, 2] - rt00, S[2, 2]])
    trS = np.trace(S)
    v = 2.0 * np.sqrt(1.0 + trS - M00 - M11 - M22)
    esii = float(np.sign(S[idx, idx]))
    r, nt = np.sqrt(2.0 + trS + v), np.sqrt(2.0 + trS - v)
    n1, n2 = np1 / np.linalg.norm(np1), np2 / np.linalg.norm(np2)
    half_nt, esii_r = 0.5 * nt, esii * r
    t1s = half_nt * (esii_r * n2 - nt * n1)
    t2s = half_nt * (esii_r * n1 - nt * n2)
    R1 = Hn @ (np.eye(3) - (2.0 / v) * np.outer(t1s, n1))
    R2 = Hn @ (np.eye(3) - (2.0 / v) * np.outer(t2s, n2))
    t1, t2 = R1 @ t1s, R2 @ t2s
    return [(R1, t1), (R1, -t1), (R2, t2), (R2, -t2)]


def triangulate(R, t, x1, x2):
    """TriangulatePoint with P1 = [I|0], P2 = [R|t] for every correspondence: the right singular vector of the
    smallest singular value of the 4 x 4 DLT matrix, by a batched SVD of A itself."""
    n = x1.shape[0]
    P2 = np.c_[R, t]
    A = np.zeros((n, 4, 4))
    A[:, 0, 0] = A[:, 1, 1] = -1.0
    A[:, 0, 2], A[:, 1, 2] = x1[:, 0], x1[:, 1]
    A[:, 2] = x2[:, :1] * P2[2] - P2[0]
    A[:, 3] = x2[:, 1:] * P2[2] - P2[1]
    if n == 0:
        return np.zeros((0, 3))
    v = np.linalg.svd(A)[2][:, -1]
    with np.errstate(divide="ignore", invalid="ignore"):
        return v[:, :3] / v[:, 3:]


def check_cheirality(R, t, x1, x2):
    """CheckCheirality: (kept [n] bool, X [n][3], margin [n][2]).  margin = distance of each depth to the nearer
    bound of (eps, max_depth), over max_depth (inf when max_depth = 0 or the depth is not a number): a
    correspondence whose margin is tiny can change sides with the rounding of another DLT solver."""
    max_depth = 1000.0 * np.linalg.norm(R.T @ t)
    X = triangulate(R, t, x1, x2)
    d1 = X[:, 2]
    d2 = (X @ R[2] + t[2]) * np.linalg.norm(R[:, 2])
    with np.errstate(invalid="ignore"):
        kept = (d1 > EPS) & (d1 < max_depth) & (d2 > EPS) & (d2 < max_depth)
        with np.errstate(divide="ignore"):
            margin = np.stack([np.minimum(np.abs(d - EPS), np.abs(max_depth - d)) / max_depth for d in (d1, d2)], 1)
    margin[~np.isfinite(margin)] = np.inf
    return kept, X, margin


def rotation_matrix_to_quaternion(R):
    """Eigen's Quaterniond(Matrix3d), returned as (w, x, y, z)."""
    R = np.asarray(R, np.float64)
    tr = R[0, 0] + R[1, 1] + R[2, 2]
    q = np.zeros(4)
    if tr > 0:
        s = np.sqrt(tr + 1.0)
        q[0] = 0.5 * s
        s = 0.5 / s
        q[1], q[2], q[3] = (R[2, 1] - R[1, 2]) * s, (R[0, 2] - R[2, 0]) * s, (R[1, 0] - R[0, 1]) * s
        return q
    i = 0
    if R[1, 1] > R[0, 0]:
        i = 1
    if R[2, 2] > R[i, i]:
        i = 2
    j, k = (i + 1) % 3, (i + 2) % 3
    s = np.sqrt(R[i, i] - R[j, j] - R[k, k] + 1.0)
    q[1 + i] = 0.5 * s
    s = 0.5 / s
    q[0] = (R[k, j] - R[j, k]) * s
    q[1 + j] = (R[j, i] + R[i, j]) * s
    q[1 + k] = (R[k, i] + R[i, k]) * s
    return q


def median(x):
    """COLMAP Median: the middle element, or the mean of the n/2-th order statistic and the largest of the lower half."""
    s = np.sort(np.asarray(x, np.float64))
    m = s.shape[0] // 2
    return float(s[m]) if s.shape[0] % 2 else float((s[m] + s[m - 1]) / 2.0)


def estimate_relative_pose(config, E, F, H, cam1, cam2, xy1, xy2):
    """EstimateRelativePose of one pair.  xy1, xy2: [n][2] keypoint locations of the inlier matches (pixels).
    Returns a dict: estimated, config, R, t, qvec, tri_angle, num_points3D, candidate, counts [ncand],
    kept [n][ncand], margin [n][ncand][2]."""
    config = int(config)
    out = dict(estimated=False, config=config, R=np.zeros((3, 3)), t=np.zeros(3), qvec=np.zeros(4), tri_angle=0.0,
               num_points3D=0, candidate=-1, counts=np.zeros(0, np.int64), kept=np.zeros((len(xy1), 0), bool),
               margin=np.zeros((len(xy1), 0, 2)))
    if config not in ESTIMATED_CONFIGS:
        return out
    x1, x2 = image_to_world(cam1, xy1), image_to_world(cam2, xy2)
    K1, K2 = calibration(cam1), calibration(cam2)
    if config in (CALIBRATED, UNCALIBRATED):
        E = np.asarray(E, np.float64).reshape(3, 3)
        if config == UNCALIBRATED:
            E = K2.T @ np.asarray(F, np.float64).reshape(3, 3) @ K1
        cands = decompose_essential_matrix(E)
    else:
        cands = decompose_homography_matrix(np.asarray(H, np.float64).reshape(3, 3), K1, K2)
    res = [check_cheirality(R, t, x1, x2) for R, t in cands]
    counts = np.array([int(k.sum()) for k, _, _ in res], np.int64)
    best = -1
    if config in (CALIBRATED, UNCALIBRATED):                # PoseFromEssentialMatrix: >=, the later candidate wins
        best, cur = 0, 0
        for i, c in enumerate(counts):
            if c >= cur:
                best, cur = i, c
    else:                                                   # PoseFromHomographyMatrix: >, non-empty only
        cur = 0
        for i, c in enumerate(counts):
            if c > 0 and c > cur:
                best, cur = i, c
        if best < 0:
            best = 0
    R, t = cands[best]
    kept, X, _ = res[best]
    Xk = X[kept]
    tri = median(triangulation_angle(np.zeros(3), -R.T @ t, Xk)) if Xk.shape[0] else 0.0
    if config == PLANAR_OR_PANORAMIC:
        if np.linalg.norm(t) == 0:
            config, tri = PANORAMIC, 0.0
        else:
            config = PLANAR
    out.update(estimated=True, config=config, R=R, t=t, qvec=rotation_matrix_to_quaternion(R), tri_angle=tri,
               num_points3D=int(counts[best]), candidate=best, counts=counts,
               kept=np.stack([k for k, _, _ in res], 1), margin=np.stack([m for _, _, m in res], 1))
    return out


def estimate_relative_poses(keypoint_ptr, keypoints, image_camera, cameras, pair_images, config, E, F, H,
                            inlier_ptr, inlier_matches):
    """Every pair of the flat arrays of init_geometry.estimate_relative_poses; returns the list of per-pair dicts."""
    out = []
    for p in range(len(config)):
        a, b = (int(v) for v in pair_images[p])
        m = np.asarray(inlier_matches[inlier_ptr[p]:inlier_ptr[p + 1]], np.int64).reshape(-1, 2)
        xy1 = keypoints[keypoint_ptr[a] + m[:, 0]]
        xy2 = keypoints[keypoint_ptr[b] + m[:, 1]]
        out.append(estimate_relative_pose(config[p], E[p], F[p], H[p], cameras[image_camera[a]],
                                          cameras[image_camera[b]], xy1, xy2))
    return out
