"""Batched (SoA) mirror of the reference's sequential point tracker around HP1.

Reference (SURVEY.md §8a rows a1, a2):
  track_optimize                      point_trajectory/track_optimize.py:24-54
  IncrementalTrajectorySet            point_trajectory/trajectory.py:98-194
      new_traj_all :117, get_cur_pos :122, extend_all :129, clear_active :154,
      optimize_buffer :161-194
  step_forward                        point_trajectory/trajectory.py:45-62
  grid_sample                         point_trajectory/trajectory.py:25-37
  flow_check / get_occ_mask           point_trajectory/utils.py:85-105

The reference keeps one Python/pybind `Trajectory` object per particle and walks them in
Python loops (≈5 pybind calls per trajectory per frame).  Here the live particles are
struct-of-arrays: per time step one [n, 2] array of locations plus index arrays that link
a particle to its slot in the two previous time steps (the 3-frame FIFO buffer of the
reference is exactly "the last three time steps").  The per-frame work is vectorised and
the optimiser is called once per frame on the whole batch, like the reference does.

Semantics that decide the INTEGER TRACK CONNECTIVITY are kept bit-for-bit:
  * flows / occlusion maps are sampled with torch.nn.functional.grid_sample on the CPU in
    float32 with the reference's normalisation (x /= (W-1)/2, -= 1; align_corners=True),
  * a particle survives iff 0 < x < W-1, 0 < y < H-1 and the sampled occlusion <= 0.1,
  * re-seeding: occupancy at (int(y), int(x)), Euclidean distance transform > ratio on the
    ratio-strided grid,
  * trajectory ids are the positions in the reference's `full_trajs` list (retire order).

track mirrors point_trajectory/track.py:24-50, the same loop without path consistency (no buffer, no HP1);
track_device runs it resident on the GPU.

track_optimize_device / main_connect_point_trajectories_device run the same loop with every particle array
resident on the GPU (csrc/tracker.cu, psfm_tracker_*) and return a TrackArrays; DESIGN.md §4.1.
"""
import ctypes as _C

import numpy as np


# ----------------------------------------------------------------------------- device ops (csrc/tracker.cu)

def _f32p(a):
    return a.ctypes.data_as(_C.POINTER(_C.c_float))


def _u8p(a):
    return a.ctypes.data_as(_C.POINTER(_C.c_uint8))


def grid_sample_device(map_hwc, xy):
    """grid_sample (trajectory.py:25-37) on the GPU, bit for bit what torch's CPU kernel returns.
    map_hwc: [H, W, C] float32 (C = 1 or 2) or [H, W]; xy [N, 2] float64 -> [N, C] float32."""
    from . import _lib
    m = np.ascontiguousarray(map_hwc, np.float32)
    if m.ndim == 2:
        m = m[:, :, None]
    h, w, c = m.shape
    xy = np.ascontiguousarray(xy, np.float64).reshape(-1, 2)
    out = np.empty((xy.shape[0], c), np.float32)
    _lib.check(_lib.lib().psfm_grid_sample(_f32p(m), h, w, c, _lib.dptr(xy), xy.shape[0], _f32p(out)), "psfm_grid_sample")
    return out


def flow_check_device(flows, flows_b, thres):
    """flow_check (point_trajectory/utils.py:58-105) on the GPU -> (error_maps, occ_maps)."""
    from . import _lib
    error_maps, occ_maps = [], []
    for f, f_b in zip(flows, flows_b):
        f = np.ascontiguousarray(f, np.float32)
        f_b = np.ascontiguousarray(f_b, np.float32)
        h, w = f.shape[:2]
        err = np.empty((h, w), np.float32)
        occ = np.empty((h, w), np.uint8)
        _lib.check(_lib.lib().psfm_flow_check(_f32p(f), _f32p(f_b), h, w, float(thres), _f32p(err), _u8p(occ)), "psfm_flow_check")
        error_maps.append(err)
        occ_maps.append(occ.astype(bool))
    return error_maps, occ_maps


def tracker_step_device(flow, occ, cur_xy, sample_ratio):
    """step_forward + the re-seeding mask of extend_all -> (next_xy, flags, reseed_mask or None)."""
    from . import _lib
    flow = np.ascontiguousarray(flow, np.float32)
    occ8 = np.ascontiguousarray(occ, np.uint8)
    h, w = flow.shape[:2]
    cur = np.ascontiguousarray(cur_xy, np.float64).reshape(-1, 2)
    n = cur.shape[0]
    nxt = np.empty((n, 2), np.float64)
    flags = np.zeros(n, np.uint8)
    gh, gw = -(-h // sample_ratio), -(-w // sample_ratio)
    mask = np.zeros((gh, gw), np.uint8)
    _lib.check(_lib.lib().psfm_tracker_step(_f32p(flow), _u8p(occ8), h, w, _lib.dptr(cur), n, sample_ratio, _lib.dptr(nxt),
                                            _u8p(flags), _u8p(mask)), "psfm_tracker_step")
    return nxt, flags, (mask.astype(bool) if flags.any() else None)


def buffer_inputs_device(flow01, flow02, occ02, x0, upper_flow=20.0):
    """optimize_buffer's ref1, ref2, scale (trajectory.py:171-183) on the GPU."""
    from . import _lib
    f1 = np.ascontiguousarray(flow01, np.float32)
    f2 = np.ascontiguousarray(flow02, np.float32)
    o2 = np.ascontiguousarray(occ02, np.uint8)
    h, w = f1.shape[:2]
    x0 = np.ascontiguousarray(x0, np.float64).reshape(-1, 2)
    n = x0.shape[0]
    ref1, ref2, scale = np.empty((n, 2)), np.empty((n, 2)), np.empty((n, 1))
    _lib.check(_lib.lib().psfm_tracker_buffer_inputs(_f32p(f1), _f32p(f2), _u8p(o2), h, w, _lib.dptr(x0), n, float(upper_flow),
                                                     _lib.dptr(ref1), _lib.dptr(ref2), _lib.dptr(scale)), "psfm_tracker_buffer_inputs")
    return ref1, ref2, scale


def grid_sample(data, xy):
    """data: torch tensor [C, H, W]; xy: [N, 2] float64 → [N, C] float32 numpy.
    Same arithmetic as point_trajectory/trajectory.py:25-37."""
    import torch
    data = data.unsqueeze(0)
    g = torch.from_numpy(np.ascontiguousarray(xy)).float().to(data.device)
    g = g.unsqueeze(0).unsqueeze(0)
    H, W = data.shape[2], data.shape[3]
    g[:, :, :, 0] /= ((W - 1) / 2)
    g[:, :, :, 1] /= ((H - 1) / 2)
    g -= 1
    out = torch.nn.functional.grid_sample(data, g, align_corners=True)
    return out.squeeze(0).squeeze(1).permute(1, 0).cpu().numpy()


def flow_check(flows, flows_b, thres):
    """Forward/backward consistency → (error_maps, occ_maps); point_trajectory/utils.py:58-105."""
    import torch
    import torch.nn.functional as F
    error_maps, occ_maps = [], []
    for f, f_b in zip(flows, flows_b):
        f_t = torch.from_numpy(f).permute(2, 0, 1).unsqueeze(0).float()
        b_t = torch.from_numpy(f_b).permute(2, 0, 1).unsqueeze(0).float()
        B, _, H, W = f_t.shape
        hh, ww = torch.meshgrid(torch.arange(H).float(), torch.arange(W).float(), indexing="ij")
        coord = torch.stack([ww, hh], 0).unsqueeze(0)
        grid = coord + f_t
        oob = ((grid[:, 0] < 0) + (grid[:, 0] > W - 1) + (grid[:, 1] < 0) + (grid[:, 1] > H - 1)).float()
        grid = grid.clone()
        grid[:, 0] /= (W - 1) / 2
        grid[:, 1] /= (H - 1) / 2
        grid -= 1
        warp = F.grid_sample(b_t, grid.permute(0, 2, 3, 1), align_corners=True)
        err = torch.norm(warp + f_t, dim=1)
        mask = torch.clamp((err > thres) + oob, 0, 1) > 0
        error_maps.append(err.squeeze().numpy())
        occ_maps.append(mask.squeeze().numpy())
    return error_maps, occ_maps


class BatchedTrajectorySet:
    """SoA replacement of IncrementalTrajectorySet (buffer_size = 3)."""

    def __init__(self, total_length, img_h, img_w, sample_ratio, optimize_fn):
        self.total_length, self.h, self.w, self.ratio = total_length, img_h, img_w, sample_ratio
        self.optimize_fn = optimize_fn
        x, y = np.arange(0, img_w), np.arange(0, img_h)
        xx, yy = np.meshgrid(x, y)
        self.all_candidates = np.stack([xx, yy], -1)[::sample_ratio, ::sample_ratio, :]
        self.sample_candidates = np.reshape(np.copy(self.all_candidates), (-1, 2))
        # per time step: ids [n] and locations [n, 2] of the particles alive at that time
        self.ids_at, self.xy_at = {}, {}
        # live particles (in the reference's active_trajs order)
        self.act_id = np.zeros(0, np.int64)
        self.act_len = np.zeros(0, np.int64)            # observations so far
        self.act_i0 = np.zeros(0, np.int64)             # slot in the current time step's arrays
        self.act_im1 = np.zeros(0, np.int64)            # slot one step back (-1: none)
        self.act_im2 = np.zeros(0, np.int64)            # slot two steps back (-1: none)
        self.next_id = 0
        self.cur_time = None
        self.retired = []                               # arrays of ids in retire order
        self.start_time = {}

    # -- new_traj_all (trajectory.py:117-120)
    def new_traj_all(self, time, points):
        n = points.shape[0]
        ids = np.arange(self.next_id, self.next_id + n, dtype=np.int64)
        self.next_id += n
        pts = points.astype(np.float64)
        if time in self.ids_at:
            base = self.ids_at[time].shape[0]
            self.ids_at[time] = np.concatenate([self.ids_at[time], ids])
            self.xy_at[time] = np.concatenate([self.xy_at[time], pts])
        else:
            base = 0
            self.ids_at[time], self.xy_at[time] = ids, pts
        self.act_id = np.concatenate([self.act_id, ids])
        self.act_len = np.concatenate([self.act_len, np.ones(n, np.int64)])
        self.act_i0 = np.concatenate([self.act_i0, base + np.arange(n, dtype=np.int64)])
        self.act_im1 = np.concatenate([self.act_im1, np.full(n, -1, np.int64)])
        self.act_im2 = np.concatenate([self.act_im2, np.full(n, -1, np.int64)])
        self.cur_time = time

    # -- get_cur_pos (trajectory.py:122-127)
    def get_cur_pos(self):
        return self.xy_at[self.cur_time][self.act_i0]

    # -- extend_all (trajectory.py:129-152)
    def extend_all(self, next_xys, next_time, flags):
        assert len(next_xys) == self.act_id.shape[0] == len(flags)
        keep = np.asarray(flags) != 0
        self.retired.append(self.act_id[~keep])
        nx = next_xys[keep]
        n = int(keep.sum())
        self.ids_at[next_time], self.xy_at[next_time] = self.act_id[keep], nx.astype(np.float64)
        self.act_id = self.act_id[keep]
        self.act_len = self.act_len[keep] + 1
        self.act_im2 = self.act_im1[keep]
        self.act_im1 = self.act_i0[keep]
        self.act_i0 = np.arange(n, dtype=np.int64)
        self.cur_time = next_time
        import scipy.ndimage
        occupied = np.zeros((self.h, self.w, 1))
        occupied[nx[:, 1].astype(np.int64), nx[:, 0].astype(np.int64)] = 1      # int() truncation
        dist = scipy.ndimage.distance_transform_edt(1.0 - occupied)
        sample_map = (dist > self.ratio)[::self.ratio, ::self.ratio, 0]
        self.sample_candidates = np.copy(self.all_candidates[sample_map])

    def clear_active(self):
        self.retired.append(self.act_id)
        self.act_id = np.zeros(0, np.int64)

    # -- optimize_buffer (trajectory.py:161-194)
    def optimize_buffer(self, flow01_map, flow12_map, flow02_map, occ02_map, next_time, upper_flow=20.0):
        import torch
        sel = np.nonzero(self.act_len >= 3)[0]          # len(buffer_xys) == 3
        t2, t1, t0 = next_time, next_time - 1, next_time - 2
        i2, i1, i0 = self.act_i0[sel], self.act_im1[sel], self.act_im2[sel]
        x0 = self.xy_at[t0][i0]
        x1 = self.xy_at[t1][i1]
        x2 = self.xy_at[t2][i2]
        if sel.shape[0] == 0:
            raise ValueError("need at least one array to stack")     # np.stack([]) in the reference
        h, w = flow01_map.shape[0], flow01_map.shape[1]
        flow01 = grid_sample(torch.from_numpy(flow01_map).permute(2, 0, 1).float(), x0)
        flow02 = grid_sample(torch.from_numpy(flow02_map).permute(2, 0, 1).float(), x0)
        occ02 = grid_sample(torch.from_numpy(occ02_map).unsqueeze(0).float(), x0)
        scale = (1.0 - occ02) * (np.linalg.norm(flow02, axis=-1, keepdims=True) < upper_flow)
        ref1 = x0 + flow01
        ref2 = x0 + flow02
        uv12 = np.concatenate([x1, x2], axis=1)
        new = self.optimize_fn(uv12, ref1, ref2, scale, flow12_map, uv12.shape[0], w, h)
        new = np.asarray(new, np.float64).reshape(-1, 2, 2)
        self.xy_at[t1][i1] = new[:, 0]
        self.xy_at[t2][i2] = new[:, 1]

    # -- results, in the reference's `full_trajs` order
    def full_trajs(self, traj_min_len=0):
        order = np.concatenate(self.retired) if self.retired else np.zeros(0, np.int64)
        rank = np.empty(self.next_id, np.int64)
        rank[order] = np.arange(order.shape[0])
        times = sorted(self.ids_at)
        ids = np.concatenate([self.ids_at[t] for t in times])
        tt = np.concatenate([np.full(self.ids_at[t].shape[0], t, np.int64) for t in times])
        xy = np.concatenate([self.xy_at[t] for t in times])
        key = np.lexsort((tt, rank[ids]))
        ids, tt, xy = rank[ids][key], tt[key], xy[key]
        bounds = np.flatnonzero(np.diff(ids)) + 1
        starts = np.concatenate([[0], bounds])
        ends = np.concatenate([bounds, [ids.shape[0]]])
        out = {}
        for s, e in zip(starts, ends):
            if e - s >= traj_min_len:
                out[int(ids[s])] = {"frame_ids": tt[s:e].tolist(), "locations": [xy[k].copy() for k in range(s, e)],
                                    "labels": [False] * int(e - s)}
        return out


class TrackArrays:
    """The track set in the reference's `full_trajs` order as four arrays: trajectory k has id ids[k] and owns
    observations ptr[k] .. ptr[k + 1] of frame_ids / xy, in time order.
        ids [T] int64, ptr [T + 1] int64, frame_ids [M] int32, xy [M, 2] float64
    labels [M] bool marks the observations the motion segmentation found dynamic; None: all static."""

    def __init__(self, ids, ptr, frame_ids, xy, labels=None):
        self.ids, self.ptr, self.frame_ids, self.xy, self.labels = ids, ptr, frame_ids, xy, labels

    def lengths(self):
        return np.diff(self.ptr)

    def to_dict(self):
        """{traj_id: {"frame_ids", "locations", "labels"}}, exactly what BatchedTrajectorySet.full_trajs returns."""
        frames = self.frame_ids.tolist()
        rows = list(self.xy.copy())             # one 1-D float64 array per location, none aliasing self.xy
        ptr = self.ptr.tolist()
        out = {}
        for k, i in enumerate(self.ids.tolist()):
            s, e = ptr[k], ptr[k + 1]
            out[i] = {"frame_ids": frames[s:e], "locations": rows[s:e],
                      "labels": [False] * (e - s) if self.labels is None else self.labels[s:e].tolist()}
        return out


def _default_optimize():
    from . import traj
    return traj.optimize_location


def track_optimize(flows, flows_f2, occ_maps, occ_maps_s2, sample_ratio, optimize_fn=None, traj_min_len=0, device=False):
    """Sequentially track and optimise point trajectories (track_optimize.py:24-54).
    Returns {traj_id: {"frame_ids", "locations", "labels"}} with the reference's ids
    (= positions in its `full_trajs` list); `traj_min_len` applies the filter of
    main_connect_point_trajectories.py:57-60.  device=True: the whole stage runs resident on the GPU
    (track_optimize_device, same bits)."""
    if device:
        return track_optimize_device(flows, flows_f2, occ_maps, occ_maps_s2, sample_ratio, optimize_fn, traj_min_len).to_dict()
    import torch
    optimize_fn = optimize_fn or _default_optimize()
    n_flows = len(flows)
    h, w = flows[0].shape[:2]
    trajs = BatchedTrajectorySet(n_flows + 1, h, w, sample_ratio, optimize_fn)
    for frame_id in range(n_flows):
        trajs.new_traj_all(frame_id, trajs.sample_candidates)
        cur_xys = trajs.get_cur_pos()
        flow_sample = grid_sample(torch.from_numpy(flows[frame_id]).permute(2, 0, 1).float(), cur_xys)
        # step_forward (trajectory.py:45-62)
        occ = grid_sample(torch.from_numpy(occ_maps[frame_id]).unsqueeze(0).float(), cur_xys) > 0.1
        next_xys = cur_xys + flow_sample
        valid = (next_xys[:, 0] > 0) * (next_xys[:, 0] < w - 1) * (next_xys[:, 1] > 0) * (next_xys[:, 1] < h - 1)
        flags = valid * (1.0 - np.squeeze(occ, axis=-1))
        trajs.extend_all(next_xys, frame_id + 1, flags)
        if frame_id + 1 >= 2:
            trajs.optimize_buffer(flows[frame_id - 1], flows[frame_id], flows_f2[frame_id - 1],
                                  occ_maps_s2[frame_id - 1], frame_id + 1)
    trajs.clear_active()
    return trajs.full_trajs(traj_min_len)


def track(flows, occ_maps, sample_ratio, traj_min_len=0, device=False):
    """Sequentially track point trajectories without path consistency (track.py:24-50): track_optimize with a
    trajectory set of buffer_size 0, so no optimize_buffer, and a frame without survivors is not an error.  The
    motion-boundary mask the reference computes there is not used by its step_forward (trajectory.py:61).  Same
    result type and ids as track_optimize; device=True: track_device(...).to_dict(), same bits."""
    if device:
        return track_device(flows, occ_maps, sample_ratio, traj_min_len).to_dict()
    import torch
    n_flows = len(flows)
    h, w = flows[0].shape[:2]
    trajs = BatchedTrajectorySet(n_flows + 1, h, w, sample_ratio, None)
    for frame_id in range(n_flows):
        trajs.new_traj_all(frame_id, trajs.sample_candidates)
        cur_xys = trajs.get_cur_pos()
        flow_sample = grid_sample(torch.from_numpy(flows[frame_id]).permute(2, 0, 1).float(), cur_xys)
        occ = grid_sample(torch.from_numpy(occ_maps[frame_id]).unsqueeze(0).float(), cur_xys) > 0.1
        next_xys = cur_xys + flow_sample
        valid = (next_xys[:, 0] > 0) * (next_xys[:, 0] < w - 1) * (next_xys[:, 1] > 0) * (next_xys[:, 1] < h - 1)
        trajs.extend_all(next_xys, frame_id + 1, valid * (1.0 - np.squeeze(occ, axis=-1)))
    trajs.clear_active()
    return trajs.full_trajs(traj_min_len)


def main_connect_point_trajectories(flows_f, flows_b, flows_f2, flows_b2, sample_ratio=2, flow_check_thres=1.0,
                                    traj_min_len=3, optimize_fn=None, device=False):
    """In-memory equivalent of main_connect_point_trajectories.py:27-62 with
    skip_path_consistency=False: returns the dict a `particlesfm.TrajectorySet` is built
    from (and np.save'd as track.npy).  device=True: main_connect_point_trajectories_device(...).to_dict()."""
    if device:
        return main_connect_point_trajectories_device(flows_f, flows_b, flows_f2, flows_b2, sample_ratio, flow_check_thres,
                                                      traj_min_len, optimize_fn).to_dict()
    _, occ = flow_check(flows_f, flows_b, flow_check_thres)
    _, occ2 = flow_check(flows_f2, flows_b2, flow_check_thres)
    return track_optimize(flows_f, flows_f2, occ, occ2, sample_ratio, optimize_fn, traj_min_len)


# ----------------------------------------------------------------------------- the stage resident on the GPU

def _on_device(a, dtype):
    """A map as a contiguous CUDA tensor of `dtype` (torch.float32 flows, torch.uint8 occlusion maps).  A numpy
    array crosses the bus here, once; a CUDA tensor of the right type is used in place."""
    import torch
    if not isinstance(a, torch.Tensor):
        a = np.ascontiguousarray(a)
        a = torch.from_numpy(a.view(np.uint8) if a.dtype == np.bool_ else a)
    if a.dtype == torch.bool and dtype == torch.uint8:
        a = a.contiguous().view(torch.uint8)
    return a.to(device="cuda", dtype=dtype).contiguous()


def _on_host(a):
    import torch
    return a.cpu().numpy() if isinstance(a, torch.Tensor) else a


class _ResidentTracker:
    """A psfm_tracker handle (csrc/tracker.cu) on torch's current stream; path_consistency=False: the mode of
    track.py (no buffer, no HP1)."""

    def __init__(self, h, w, sample_ratio, num_frames, path_consistency=True):
        from . import _lib
        self.L, self.check = _lib.lib(), _lib.check
        self.h, self.w, self.num_frames = h, w, num_frames
        self.path_consistency = path_consistency
        self.occ = self.occ2 = None             # advance()'s occlusion maps, reused frame after frame
        self.handle = _C.c_void_p()
        self.stream = None
        if self.L.psfm_device_count() > 0:      # without a device the library refuses below, before torch touches CUDA
            import torch
            self.stream = torch.cuda.current_stream().cuda_stream
        if path_consistency:
            self.check(self.L.psfm_tracker_create(h, w, sample_ratio, num_frames, self.stream, _C.byref(self.handle)),
                       "psfm_tracker_create")
        else:
            self.check(self.L.psfm_tracker_create_mode(h, w, sample_ratio, num_frames, 0, self.stream, _C.byref(self.handle)),
                       "psfm_tracker_create_mode")

    def close(self):
        if self.handle:
            self.L.psfm_tracker_destroy(self.handle)
            self.handle = _C.c_void_p()

    def flow_check(self, flow_f, flow_b, thres, out=None):
        import torch
        occ = torch.empty((self.h, self.w), dtype=torch.uint8, device=flow_f.device) if out is None else out
        self.check(self.L.psfm_flow_check_device(flow_f.data_ptr(), flow_b.data_ptr(), self.h, self.w, float(thres), None,
                                                 occ.data_ptr(), self.stream), "psfm_flow_check_device")
        return occ

    def step(self, flow, occ, flow_prev=None, flow2_prev=None, occ2_prev=None):
        """new_traj_all + step_forward + extend_all (+ optimize_buffer's selection) -> number of buffered particles"""
        ptr = lambda t: None if t is None else t.data_ptr()
        counts = (_C.c_int32 * 3)()
        self.check(self.L.psfm_tracker_advance(self.handle, flow.data_ptr(), occ.data_ptr(), ptr(flow_prev), ptr(flow2_prev),
                                               ptr(occ2_prev), counts), "psfm_tracker_advance")
        return counts[2]

    def optimize_buffer(self, n, optimize_fn, flow12_map):
        if n == 0:
            raise ValueError("need at least one array to stack")     # np.stack([]) in the reference
        if optimize_fn is None:
            self.check(self.L.psfm_tracker_optimize(self.handle, None, None), "psfm_tracker_optimize")
            return
        from . import _lib
        uv12, ref1, ref2, scale = np.empty((n, 4)), np.empty((n, 2)), np.empty((n, 2)), np.empty((n, 1))
        self.check(self.L.psfm_tracker_get_buffer(self.handle, _lib.dptr(uv12), _lib.dptr(ref1), _lib.dptr(ref2),
                                                  _lib.dptr(scale)), "psfm_tracker_get_buffer")
        new = optimize_fn(uv12, ref1, ref2, scale, _on_host(flow12_map), n, self.w, self.h)
        new = np.ascontiguousarray(np.asarray(new, np.float64).reshape(n, 4))
        self.check(self.L.psfm_tracker_set_buffer(self.handle, _lib.dptr(new)), "psfm_tracker_set_buffer")

    def advance(self, t, flow_f, flow_b, flow_prev=None, flow_f2=None, flow_b2=None, thres=1.0, optimize_fn=None,
                flow12_map=None):
        """Frame t of main_connect_point_trajectories.py: the flow check of pair (t, 1) (flow_f, flow_b), with path
        consistency from t = 1 on the flow check of pair (t-1, 2) (flow_f2, flow_b2), the step (flow_prev: the
        forward map of pair (t-1, 1)) and optimize_buffer (optimize_fn None: HP1 on the device; otherwise it gets
        flow12_map, default flow_f, as optimize_buffer gives it).  Maps are CUDA tensors on the tracker's stream;
        they may be dropped once this returns, as the stream orders any reuse of their memory after this work."""
        import torch
        if self.occ is None:
            self.occ = torch.empty((self.h, self.w), dtype=torch.uint8, device=flow_f.device)
        self.flow_check(flow_f, flow_b, thres, out=self.occ)
        if self.path_consistency and t >= 1:
            if self.occ2 is None:
                self.occ2 = torch.empty((self.h, self.w), dtype=torch.uint8, device=flow_f.device)
            self.flow_check(flow_f2, flow_b2, thres, out=self.occ2)
            n = self.step(flow_f, self.occ, flow_prev, flow_f2, self.occ2)
            self.optimize_buffer(n, optimize_fn, flow_f if flow12_map is None else flow12_map)
        else:
            self.step(flow_f, self.occ)

    def finish(self, traj_min_len, result=True):
        """psfm_tracker_finish -> the track set's TrackArrays (host copies); result=False: (number of trajectories,
        number of observations) only, the set left on the device for matches() and track_npy_body()."""
        from . import _lib
        nt, m = _C.c_int64(), _C.c_int64()
        self.check(self.L.psfm_tracker_finish(self.handle, int(traj_min_len), _C.byref(nt), _C.byref(m)), "psfm_tracker_finish")
        if not result:
            return nt.value, m.value
        ids, ptr = np.empty(nt.value, np.int64), np.empty(nt.value + 1, np.int64)
        frame_ids, xy = np.empty(m.value, np.int32), np.empty((m.value, 2), np.float64)
        i64 = lambda a: a.ctypes.data_as(_C.POINTER(_C.c_int64))
        self.check(self.L.psfm_tracker_result(self.handle, i64(ids), i64(ptr), frame_ids.ctypes.data_as(_C.POINTER(_C.c_int32)),
                                              _lib.dptr(xy)), "psfm_tracker_result")
        return TrackArrays(ids, ptr, frame_ids, xy)

    def matches(self, num_images, sample_k):
        """After finish(): psfm_tracker_matches, the hand-off's psfm_matches handle built from the track set where it
        lies -> (handle, number of ordered pairs, number of matches); the caller destroys the handle."""
        handle, npairs, nmatches = _C.c_void_p(), _C.c_int64(), _C.c_int64()
        self.check(self.L.psfm_tracker_matches(self.handle, int(num_images), int(sample_k), _C.byref(handle),
                                               _C.byref(npairs), _C.byref(nmatches)), "psfm_tracker_matches")
        return handle, npairs.value, nmatches.value

    def track_npy_body(self):
        """After finish(): the finished track set's track.npy state body, encoded on the device where the set lies
        (csrc/track_npy.cu) -> a TrackNpyBody."""
        body = TrackNpyBody()
        self.check(self.L.psfm_tracker_track_npy(self.handle, _C.byref(body.handle), _C.byref(body.nbytes)),
                   "psfm_tracker_track_npy")
        return body


class TrackNpyBody:
    """The bytes of a track.npy state body in a pinned host buffer the library owns; view() is valid until close()."""

    def __init__(self):
        from . import _lib
        self.L = _lib.lib()
        self.handle, self.nbytes = _C.c_void_p(), _C.c_int64()

    def view(self):
        n = self.nbytes.value
        return memoryview((_C.c_uint8 * n).from_address(self.L.psfm_track_npy_data(self.handle))).cast("B")

    def close(self):
        if self.handle:
            self.L.psfm_track_npy_destroy(self.handle)
            self.handle = _C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def track_npy_body_device(arrays):
    """The track.npy state body of any TrackArrays (host arrays, uploaded), encoded by csrc/track_npy.cu.  Ids
    outside [0, 2^31), negative frame ids and a ptr that does not run monotonically from 0 to the number of
    observations are refused (PsfmError, PSFM_ERR_INVALID) before the device is used."""
    from . import _lib
    ids = np.ascontiguousarray(arrays.ids, np.int64)
    ptr = np.ascontiguousarray(arrays.ptr, np.int64)
    frame_ids = np.ascontiguousarray(arrays.frame_ids, np.int32)
    xy = np.ascontiguousarray(arrays.xy, np.float64).reshape(-1, 2)
    if ptr.shape != (ids.shape[0] + 1,) or frame_ids.shape[0] != xy.shape[0]:
        raise ValueError("TrackArrays: ptr must have one entry more than ids, frame_ids as many as xy rows")
    i64 = lambda a: a.ctypes.data_as(_C.POINTER(_C.c_int64))
    body = TrackNpyBody()
    _lib.check(body.L.psfm_track_npy_create(i64(ids), i64(ptr), frame_ids.ctypes.data_as(_C.POINTER(_C.c_int32)), _lib.dptr(xy),
                                            ids.shape[0], frame_ids.shape[0], _C.byref(body.handle), _C.byref(body.nbytes)),
               "psfm_track_npy_create")
    return body


def track_device(flows, occ_maps, sample_ratio, traj_min_len=0):
    """track (track.py:24-50) resident on the GPU -> TrackArrays, bit for bit the host path's track set.  Maps as
    track_optimize_device takes them."""
    n_flows = len(flows)
    h, w = flows[0].shape[:2]
    trk = _ResidentTracker(h, w, sample_ratio, n_flows + 1, path_consistency=False)
    try:
        import torch
        for frame_id in range(n_flows):
            trk.step(_on_device(flows[frame_id], torch.float32), _on_device(occ_maps[frame_id], torch.uint8))
        return trk.finish(traj_min_len)
    finally:
        trk.close()


def track_optimize_device(flows, flows_f2, occ_maps, occ_maps_s2, sample_ratio, optimize_fn=None, traj_min_len=0):
    """track_optimize (track_optimize.py:24-54) resident on the GPU -> TrackArrays, bit for bit the host path's
    track set.  Maps are numpy arrays or CUDA tensors ([H, W, 2] float32 flows, [H, W] bool occlusion maps); each
    crosses the bus at most once.  optimize_fn=None: HP1 on the device; otherwise it is called per frame with host
    arrays, as optimize_buffer calls it: (uv12, ref1, ref2, scale, flow12_map, n, w, h)."""
    n_flows = len(flows)
    h, w = flows[0].shape[:2]
    trk = _ResidentTracker(h, w, sample_ratio, n_flows + 1)
    try:
        import torch
        prev = None
        for frame_id in range(n_flows):
            flow = _on_device(flows[frame_id], torch.float32)
            occ = _on_device(occ_maps[frame_id], torch.uint8)
            if frame_id + 1 >= 2:
                n = trk.step(flow, occ, prev, _on_device(flows_f2[frame_id - 1], torch.float32),
                             _on_device(occ_maps_s2[frame_id - 1], torch.uint8))
                trk.optimize_buffer(n, optimize_fn, flows[frame_id])
            else:
                trk.step(flow, occ)
            prev = flow
        return trk.finish(traj_min_len)
    finally:
        trk.close()


def main_connect_point_trajectories_device(flows_f, flows_b, flows_f2, flows_b2, sample_ratio=2, flow_check_thres=1.0,
                                           traj_min_len=3, optimize_fn=None):
    """main_connect_point_trajectories resident on the GPU -> TrackArrays: the flow check runs inside the loop on
    the resident maps, and its occlusion maps never leave the device."""
    n_flows = len(flows_f)
    h, w = flows_f[0].shape[:2]
    trk = _ResidentTracker(h, w, sample_ratio, n_flows + 1)
    try:
        import torch
        f32 = torch.float32
        prev = None
        for frame_id in range(n_flows):
            flow = _on_device(flows_f[frame_id], f32)
            f2 = b2 = None
            if frame_id >= 1:
                f2, b2 = _on_device(flows_f2[frame_id - 1], f32), _on_device(flows_b2[frame_id - 1], f32)
            trk.advance(frame_id, flow, _on_device(flows_b[frame_id], f32), prev, f2, b2, flow_check_thres, optimize_fn,
                        flows_f[frame_id])
            prev = flow
        return trk.finish(traj_min_len)
    finally:
        trk.close()
