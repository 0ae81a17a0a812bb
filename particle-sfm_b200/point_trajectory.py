"""The point-trajectory stage as a command: a flow directory in, traj_dir/track.npy out, on the GPU (DESIGN.md §4.13).

    python -m particlesfm_b200.point_trajectory --flow_dir F --traj_dir T [--sample_ratio 2] [--traj_min_len 3]
        [--flow_check_thres 1.0] [--skip_path_consistency] [--skip_exists]

Reference: point_trajectory/main_connect_point_trajectories.py:27-75 with utils.py:26-56 (load_flows, read_flo),
track.py:24-50 (--skip_path_consistency) and track_optimize.py:24-54.

The .flo files are read ahead on a host thread into pinned staging buffers and uploaded on a copy stream into a
ring of three device slots, so that frame t+1's maps cross the bus while frame t's flow check, tracker kernels and
HP1 run; the host never holds the whole sequence and the device maps do not grow with the number of frames.  The
track set stays on the device until csrc/track_npy.cu has written the body of the file's pickled state; the host
wraps it in the npy header and pickle opcodes the running numpy and pickle write for an empty TrajectorySet.
"""
import argparse
import glob
import io
import os
import pickletools
import queue
import sys
import threading

import numpy as np

from . import tracker

TAG_FLOAT = 202021.25
_HEADER = 12                    # tag, w, h
_SLOTS = 3                      # pinned staging slots and device slots


# ----------------------------------------------------------------------------- .flo files

def list_flows(d):
    """The .flo files of a directory in load_flows' order (utils.py:26-31)."""
    return sorted(glob.glob(os.path.join(d, "*.flo")))


def flo_size(path):
    """(h, w) of a .flo file whose header and length are valid: the tag 202021.25, w and h as int32, then at least
    2 * w * h float32 values (trailing bytes are ignored, as read_flo's np.fromfile(count=...) ignores them).
    ValueError naming the file otherwise."""
    size = os.path.getsize(path)
    if size < _HEADER:
        raise ValueError("%s: %d bytes, shorter than the 12-byte .flo header" % (path, size))
    with open(path, "rb") as f:
        head = f.read(_HEADER)
    tag = np.frombuffer(head, "<f4", 1)[0]
    w, h = (int(v) for v in np.frombuffer(head, "<i4", 2, 4))
    if tag != np.float32(TAG_FLOAT):
        raise ValueError("%s: tag %r is not the .flo tag %r" % (path, float(tag), TAG_FLOAT))
    if w < 2 or h < 2:
        raise ValueError("%s: size %d x %d; a flow map needs at least 2 x 2 pixels" % (path, w, h))
    if size < _HEADER + 8 * w * h:
        raise ValueError("%s: %d bytes, short of the %d a %d x %d .flo holds" % (path, size, _HEADER + 8 * w * h, w, h))
    return h, w


def read_flo(path):
    """read_flo (utils.py:38-56) of a valid file: [h, w, 2] float32; malformed files raise ValueError (flo_size)."""
    h, w = flo_size(path)
    with open(path, "rb") as f:
        f.seek(_HEADER)
        return np.fromfile(f, "<f4", 2 * w * h).astype(np.float32, copy=False).reshape(h, w, 2)


def flow_frames(flow_dir, skip_path_consistency=False):
    """Check a flow directory before anything runs and list, per frame t, the files the stage reads there:
    flow_f[t], flow_b[t], and with path consistency from t = 1 on flow_f2[t-1], flow_b2[t-1].  -> (frames, h, w).
    ValueError naming the directory or file: no flow_f map, a flow_b count other than flow_f's, fewer than
    len(flow_f) - 1 maps in flow_f2 or flow_b2 (extra ones are ignored), a malformed file, maps of different sizes."""
    sub = lambda name: os.path.join(flow_dir, name)
    ff, fb = list_flows(sub("flow_f")), list_flows(sub("flow_b"))
    if not ff:
        raise ValueError("%s: no .flo file" % sub("flow_f"))
    if len(fb) != len(ff):
        raise ValueError("%s: %d .flo files, %s has %d" % (sub("flow_b"), len(fb), sub("flow_f"), len(ff)))
    frames = [[a, b] for a, b in zip(ff, fb)]
    if not skip_path_consistency:
        for name in ("flow_f2", "flow_b2"):
            f2 = list_flows(sub(name))
            if len(f2) < len(ff) - 1:
                raise ValueError("%s: %d .flo files, path consistency needs %d" % (sub(name), len(f2), len(ff) - 1))
            for t in range(1, len(ff)):
                frames[t].append(f2[t - 1])
    shape = None
    for paths in frames:
        for p in paths:
            s = flo_size(p)
            if shape is None:
                shape = s
            elif s != shape:
                raise ValueError("%s: size %d x %d, the sequence's maps are %d x %d" % (p, s[1], s[0], shape[1], shape[0]))
    return frames, shape[0], shape[1]


class _FlowStream:
    """Frame t's maps on the device: a reader thread fills pinned staging slots (readinto releases the GIL),
    upload(t) copies them on a copy stream into device slot t % 3, maps(t) orders torch's current stream after
    that copy, release(t) lets the slot be overwritten once the current stream's work so far is done."""

    def __init__(self, frames, h, w):
        import torch
        self.frames, self.hw = frames, (h, w)
        k = max(len(p) for p in frames)
        self.host = torch.empty((_SLOTS, k, h, w, 2), dtype=torch.float32, pin_memory=True)
        self.dev = torch.empty((_SLOTS, k, h, w, 2), dtype=torch.float32, device="cuda")
        self.copy = torch.cuda.Stream()
        self.uploaded, self.dev_free = [None] * _SLOTS, [None] * _SLOTS
        self.free, self.ready = queue.Queue(), queue.Queue()
        for s in range(_SLOTS):
            self.free.put((s, None))
        self.thread = threading.Thread(target=self._read, name="psfm-flo-reader", daemon=True)
        self.thread.start()

    def _read(self):
        host = self.host.numpy()
        nbytes = 8 * self.hw[0] * self.hw[1]
        try:
            for t, paths in enumerate(self.frames):
                item = self.free.get()
                if item is None:
                    return
                s, ev = item
                if ev is not None:
                    ev.synchronize()           # the slot's previous upload has left it
                for i, p in enumerate(paths):
                    with open(p, "rb", buffering=0) as f:
                        f.seek(_HEADER)
                        got = f.readinto(memoryview(host[s, i]).cast("B"))
                    if got != nbytes:
                        raise ValueError("%s: %d bytes of flow read, %d expected" % (p, got, nbytes))
                self.ready.put((t, s))
        except BaseException as e:      # handed to the consumer, which raises it
            self.ready.put(e)

    def upload(self, t):
        import torch
        item = self.ready.get()
        if isinstance(item, BaseException):
            raise item
        _, s = item
        d, n = t % _SLOTS, len(self.frames[t])
        with torch.cuda.stream(self.copy):
            if self.dev_free[d] is not None:
                self.copy.wait_event(self.dev_free[d])
            self.dev[d, :n].copy_(self.host[s, :n], non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.copy)
        self.uploaded[d] = ev
        self.free.put((s, ev))

    def maps(self, t):
        import torch
        torch.cuda.current_stream().wait_event(self.uploaded[t % _SLOTS])
        return self.dev[t % _SLOTS]

    def release(self, t):
        import torch
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream())
        self.dev_free[t % _SLOTS] = ev

    def close(self):
        self.free.put(None)
        self.thread.join()


# ----------------------------------------------------------------------------- track.npy

def _particlesfm():
    here = os.path.dirname(os.path.abspath(__file__))
    if here not in sys.path:
        sys.path.insert(0, here)
    import particlesfm
    return particlesfm


_FRAMING = None


def npy_framing():
    """(head, tail) around the state body: np.save of an empty particlesfm.TrajectorySet, split at the EMPTY_DICT of
    its state, the length of a protocol-4 FRAME around it left to patch.  -> (head, tail, frame_len_at, frame_len)
    with frame_len_at None when the stream has no frame around the state."""
    global _FRAMING
    if _FRAMING is None:
        buf = io.BytesIO()
        np.save(buf, _particlesfm().TrajectorySet())
        raw = buf.getvalue()
        start = 10 + int.from_bytes(raw[8:10], "little") if raw[6] == 1 else 12 + int.from_bytes(raw[8:12], "little")
        ops = list(pickletools.genops(raw[start:]))
        dicts = [pos for op, _, pos in ops if op.name == "EMPTY_DICT"]
        if len(dicts) != 1:
            raise RuntimeError("np.save of an empty TrajectorySet holds %d EMPTY_DICT opcodes, expected 1" % len(dicts))
        at = start + dicts[0]
        frame = None
        for op, arg, pos in ops:
            if op.name == "FRAME" and start + pos + 9 <= at < start + pos + 9 + arg:
                frame = (start + pos + 1, arg)
        _FRAMING = (raw[:at], raw[at + 1:]) + (frame if frame else (None, None))
    return _FRAMING


def write_track_npy(path, body):
    """track.npy from a state body (bytes-like): np.load(path, allow_pickle=True).item() is the TrajectorySet.  The
    file is written beside `path` and renamed, so a failed write leaves no partial file."""
    head, tail, frame_at, frame_len = npy_framing()
    body = memoryview(body).cast("B")
    if frame_at is not None:
        head = head[:frame_at] + (frame_len - 1 + body.nbytes).to_bytes(8, "little") + head[frame_at + 8:]
    tmp = path + ".tmp"
    try:
        with open(tmp, "wb") as f:
            f.write(head)
            f.write(body)
            f.write(tail)
        os.replace(tmp, path)
    except BaseException:
        if os.path.exists(tmp):
            os.remove(tmp)
        raise


# ----------------------------------------------------------------------------- the stage

def connect_point_trajectories(flow_dir, sample_ratio=2, flow_check_thres=1.0, traj_min_len=3, skip_path_consistency=False,
                               npy_path=None):
    """The stage from a checked flow directory -> tracker.TrackArrays; with npy_path, the track set is also written
    there as track.npy from the device."""
    frames, h, w = flow_frames(flow_dir, skip_path_consistency)
    n_flows = len(frames)
    pc = not skip_path_consistency
    trk = tracker._ResidentTracker(h, w, sample_ratio, n_flows + 1, path_consistency=pc)
    stream = None
    try:
        stream = _FlowStream(frames, h, w)
        stream.upload(0)
        prev = None
        for t in range(n_flows):
            if t + 1 < n_flows:
                stream.upload(t + 1)           # crosses the bus while frame t runs
            m = stream.maps(t)
            flow = m[0]
            f2, b2 = (m[2], m[3]) if pc and t >= 1 else (None, None)
            trk.advance(t, flow, m[1], prev, f2, b2, flow_check_thres)
            if t >= 1:
                stream.release(t - 1)
            prev = flow
        arrays = trk.finish(traj_min_len)
        if npy_path is not None:
            with trk.track_npy_body() as body:
                write_track_npy(npy_path, body.view())
        return arrays
    finally:
        if stream is not None:
            stream.close()
        trk.close()


def main_connect_point_trajectories(flow_dir, traj_dir, sample_ratio=2, flow_check_thres=1.0, traj_min_len=3,
                                    skip_path_consistency=False, skip_exists=False):
    """main_connect_point_trajectories.py:27-62: traj_dir/track.npy from flow_dir's flow_f, flow_b (and flow_f2,
    flow_b2 with path consistency), traj_dir created if missing.  Returns the tracker.TrackArrays written, or None
    when skip_exists finds the file (no flow is opened then).  Malformed input raises ValueError before anything is
    written."""
    os.makedirs(traj_dir, exist_ok=True)
    out = os.path.join(traj_dir, "track.npy")
    if skip_exists and os.path.exists(out):
        return None
    return connect_point_trajectories(flow_dir, sample_ratio, flow_check_thres, traj_min_len, skip_path_consistency, out)


def main(argv=None):
    p = argparse.ArgumentParser("Connecting and optimizing point trajectories from pairwise flows")
    p.add_argument("--flow_dir", required=True, help="path to the folder of optical flows")
    p.add_argument("--traj_dir", required=True, help="trajectory output")
    p.add_argument("--sample_ratio", type=int, default=2, help="sample ratio of trajectories")
    p.add_argument("--traj_min_len", type=int, default=3, help="minimum length of the trajectories")
    p.add_argument("--flow_check_thres", type=float, default=1.0, help="flow consistency check threshold")
    p.add_argument("--skip_path_consistency", action="store_true", help="whether to skip the path consistency optimization or not")
    p.add_argument("--skip_exists", action="store_true", help="keep an existing track.npy")
    a = p.parse_args(argv)
    try:
        main_connect_point_trajectories(a.flow_dir, a.traj_dir, a.sample_ratio, a.flow_check_thres, a.traj_min_len,
                                        a.skip_path_consistency, a.skip_exists)
    except ValueError as e:
        print("point_trajectory: %s" % e, file=sys.stderr)
        return 1
    return 0


if __name__ == "__main__":
    sys.exit(main())
