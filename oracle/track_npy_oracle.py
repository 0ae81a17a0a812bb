"""Numpy encoder of track.npy's state body (TEST INFRASTRUCTURE): the bytes csrc/track_npy.cu writes, from the four
arrays of a tracker.TrackArrays, built with whole-array operations.

The body is the pickled dict {id: {"frame_ids": [...], "locations": [(x, y), ...], "labels": [False, ...]}} in
protocol-2 opcodes without memo: per trajectory its id (BININT1 / BININT2 / BININT), then
    }( X"frame_ids" ]( <frame ids> e X"locations" ]( <G x G y \\x86 per location> e X"labels" ]( <\\x89 per label> e u
and around the records }( ... u (a lone } for no trajectory)."""
import numpy as np

_U1 = np.uint8


def _key(name):
    return b"X" + len(name).to_bytes(4, "little") + name.encode()


HEAD_FRAMES = b"}(" + _key("frame_ids") + b"]("
HEAD_LOCATIONS = b"e" + _key("locations") + b"]("
HEAD_LABELS = b"e" + _key("labels") + b"]("
TAIL = b"eu"
LOCATION = 19                   # G x G y \x86


def _int_opcodes(v):
    """BININT1 / BININT2 / BININT of each non-negative v < 2^31: (widths [n], bytes [n, 5], of which widths are used)."""
    v = np.asarray(v, np.int64)
    small, mid = v < 256, v < 65536
    width = np.where(small, 2, np.where(mid, 3, 5))
    out = np.zeros((v.shape[0], 5), _U1)
    out[:, 0] = np.where(small, ord("K"), np.where(mid, ord("M"), ord("J")))
    out[:, 1:] = v.astype("<u4").view(_U1).reshape(-1, 4)
    return width, out


def _put_const(buf, starts, const):
    c = np.frombuffer(const, _U1)
    buf[starts[:, None] + np.arange(c.shape[0])] = c


def _put_ints(buf, starts, width, ops):
    pos = starts[:, None] + np.arange(5)
    used = np.arange(5) < width[:, None]
    buf[pos[used]] = ops[used]


def encode_body(ids, ptr, frame_ids, xy):
    """The body of the TrajectorySet state for trajectory k = ids[k] owning observations ptr[k] .. ptr[k + 1]."""
    ids = np.asarray(ids, np.int64)
    ptr = np.asarray(ptr, np.int64)
    frame_ids = np.asarray(frame_ids, np.int64)
    xy = np.asarray(xy, np.float64).reshape(-1, 2)
    T, M = ids.shape[0], frame_ids.shape[0]
    if ptr.shape != (T + 1,) or ptr[0] != 0 or ptr[-1] != M or xy.shape[0] != M or (np.diff(ptr) < 0).any():
        raise ValueError("ptr must run monotonically from 0 to the number of observations")
    if ((ids < 0) | (ids >= 2 ** 31)).any() or (frame_ids < 0).any():
        raise ValueError("trajectory ids must lie in [0, 2^31) and frame ids be non-negative")
    if T == 0:
        return b"}"
    L = np.diff(ptr)
    rec = np.repeat(np.arange(T), L)
    idw, idops = _int_opcodes(ids)
    fw, fops = _int_opcodes(frame_ids)
    fcum = np.concatenate([[0], np.cumsum(fw)])
    fsum = fcum[ptr[1:]] - fcum[ptr[:-1]]
    size = idw + len(HEAD_FRAMES) + fsum + len(HEAD_LOCATIONS) + LOCATION * L + len(HEAD_LABELS) + L + len(TAIL)
    start = 2 + np.concatenate([[0], np.cumsum(size)[:-1]])
    buf = np.zeros(3 + int(size.sum()), _U1)
    buf[0], buf[1], buf[-1] = ord("}"), ord("("), ord("u")
    _put_ints(buf, start, idw, idops)
    frames0 = start + idw + len(HEAD_FRAMES)
    _put_const(buf, start + idw, HEAD_FRAMES)
    _put_ints(buf, frames0[rec] + (fcum[:-1] - fcum[ptr[:-1]][rec]), fw, fops)
    lhead = frames0 + fsum
    _put_const(buf, lhead, HEAD_LOCATIONS)
    within = np.arange(M) - ptr[:-1][rec]
    loc = np.empty((M, LOCATION), _U1)
    loc[:, 0] = loc[:, 9] = ord("G")
    be = xy.astype(">f8").view(_U1).reshape(M, 2, 8)
    loc[:, 1:9], loc[:, 10:18] = be[:, 0], be[:, 1]
    loc[:, 18] = 0x86
    buf[(lhead + len(HEAD_LOCATIONS))[rec][:, None] + LOCATION * within[:, None] + np.arange(LOCATION)] = loc
    bhead = lhead + len(HEAD_LOCATIONS) + LOCATION * L
    _put_const(buf, bhead, HEAD_LABELS)
    bbase = bhead + len(HEAD_LABELS)
    buf[bbase[rec] + within] = 0x89
    _put_const(buf, bbase + L, TAIL)
    return buf.tobytes()
