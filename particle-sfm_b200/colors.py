"""The 3D points' colours from the images that observe them, on the GPU (DESIGN.md §4.11).

    python -m particlesfm_b200.colors --image_path DIR --input_path MODEL --output_path MODEL2

`extract_colors_for_all_images` is Reconstruction::ExtractColorsForAllImages (reference base/reconstruction.cc:
1250-1300), which gcolmap's global mapper runs after its refinement when GlobalMapperOptions::extract_colors is set:
every observation (a keypoint with a point) of every image that can be read is sampled bilinearly at (X - 0.5,
Y - 0.5), and each point gets the mean of its samples rounded half away from zero, or black when it has none.  The
samples are summed in a fixed order, ascending image then keypoint (the reference's order is not defined), so two
runs give the same bytes.  The command line is COLMAP's color_extractor on a binary model: it writes the model back
with only the points' rgb bytes changed.

Images are read as COLMAP's Bitmap::Read(as_rgb = true) reads them, with Pillow: modes RGB, RGBA, L, LA and P become
RGB8 through convert("RGB"), which replicates grey, drops alpha without compositing and expands palettes.  Any other
mode (16-bit, CMYK, I, F, 1) is a ValueError naming the image, raised before anything runs on the device.  A missing
or undecodable file is skipped with the reference's message, "Could not read image NAME at path PATH.".  JPEG pixels
can differ from FreeImage's by a level or so (DESIGN.md §4.11); PNG pixels are the same.

Decoding runs on a thread pool while the device samples the previous batch.  A batch is a run of consecutive read
images whose RGB8 bytes fit in half of `memory_budget` (at least one image); batch k is sampled on stream k % 2.
"""
import argparse
import collections
import concurrent.futures
import ctypes as C
import os
import sys
import time

import numpy as np

from . import _abi, _lib, colmap_io

DEVICE_BUDGET = 256 << 20          # bytes of device memory for the two batch slots' pixels
MODES = ("RGB", "RGBA", "L", "LA", "P")


class ColorsReport:
    """unread (names of the images that could not be read, in index order), images (images read), num_batches,
    num_observations (keypoints with a point), seconds {stage: s}: open (reading every image's header), setup (the
    observations' upload and sort, CUDA events), decode (decoding, summed over the threads), decode_wait (wall time
    the batches waited for the decoders), stage (copies into the pinned buffers), upload, sample, mean (CUDA events)
    and total."""

    def __init__(self):
        self.unread, self.images, self.num_batches, self.num_observations, self.seconds = [], 0, 0, 0, {}


def point_rows(point3D_ids, point_ids):
    """The row in point_ids of every keypoint's point3D_id, -1 for none; a point3D_id not in point_ids is a KeyError."""
    p3 = np.asarray(point3D_ids, np.int64)
    point_ids = np.asarray(point_ids, np.int64)
    order = np.argsort(point_ids, kind="stable")
    has = p3 != -1
    pos = np.searchsorted(point_ids[order], p3[has])
    found = pos < len(point_ids)
    found[found] = point_ids[order][pos[found]] == p3[has][found]
    if not found.all():
        raise KeyError(int(p3[has][~found][0]))
    row = np.full(len(p3), -1, np.int32)
    row[has] = order[pos]
    return row


def _header(path):
    """(mode, width, height) of the image at path, or None when Pillow cannot open it."""
    from PIL import Image
    try:
        with Image.open(path) as im:
            return im.mode, im.size[0], im.size[1]
    except OSError:
        return None


def _decode(path):
    """(RGB8 [h][w][3] or None when the file cannot be decoded, seconds)."""
    from PIL import Image
    t0 = time.perf_counter()
    try:
        with Image.open(path) as im:
            rgb = np.ascontiguousarray(im.convert("RGB"))
    except OSError:
        rgb = None
    return rgb, time.perf_counter() - t0


def extract_colors_for_all_images(image_path, image_names, keypoint_ptr, keypoints, point3D_of_keypoint, num_points,
                                  memory_budget=DEVICE_BUDGET, verbose=True, threads=None):
    """rgb [num_points][3] uint8 and a ColorsReport for the images image_names (read from image_path/NAME; names may
    hold subdirectories) with keypoint_ptr [F + 1] over keypoints [K][2] and point3D_of_keypoint [K] (point row in
    [0, num_points), -1: none).  verbose prints the reference's line for every image that cannot be read."""
    t_start = time.perf_counter()
    rep = ColorsReport()
    F = len(image_names)
    kp_ptr = np.ascontiguousarray(keypoint_ptr, np.int64)
    keypoints = np.ascontiguousarray(np.asarray(keypoints, np.float64).reshape(-1, 2))
    rows = np.ascontiguousarray(point3D_of_keypoint, np.int32)
    paths = [os.path.join(image_path, n) for n in image_names]
    threads = threads or min(32, os.cpu_count() or 1)
    rgb = np.zeros((num_points, 3), np.uint8)
    L = _lib.lib()
    s = _abi.ColorsSummary()
    i64p, ip, u8p = C.POINTER(C.c_int64), C.POINTER(C.c_int32), C.POINTER(C.c_uint8)
    with concurrent.futures.ThreadPoolExecutor(threads) as pool:
        # every image's header, so that an unsupported mode is refused before any launch
        t0 = time.perf_counter()
        heads = list(pool.map(_header, paths))
        for name, path, hd in zip(image_names, paths, heads):
            if hd is not None and hd[0] not in MODES:
                raise ValueError(f"image {name!r} at {path} has Pillow mode {hd[0]}; only 8-bit RGB, RGBA, grey, grey "
                                 f"with alpha and palette images are read")
        rep.seconds["open"] = time.perf_counter() - t0
        h = C.c_void_p()
        _lib.check(L.psfm_colors_create(F, kp_ptr.ctypes.data_as(i64p), _lib.dptr(keypoints), rows.ctypes.data_as(ip),
                                        int(num_points), C.byref(h), C.byref(s)), "psfm_colors_create")
        try:
            rep.num_observations = s.num_observations
            unread = [False] * F
            batch, batch_bytes = [], 0          # [(image, rgb8)] of consecutive read images
            decode, wait = 0.0, 0.0

            def flush():
                nonlocal batch, batch_bytes
                if not batch:
                    return
                w = np.array([a.shape[1] for _, a in batch], np.int32)
                hh = np.array([a.shape[0] for _, a in batch], np.int32)
                px = np.concatenate([a.reshape(-1) for _, a in batch])
                _lib.check(L.psfm_colors_add_images(h, batch[0][0], len(batch), w.ctypes.data_as(ip),
                                                    hh.ctypes.data_as(ip), px.ctypes.data_as(u8p)),
                           "psfm_colors_add_images")
                rep.num_batches += 1
                batch, batch_bytes = [], 0

            todo = [i for i in range(F) if heads[i] is not None]
            for i in range(F):
                unread[i] = heads[i] is None
            pending = collections.deque()
            nxt = 0
            for i in range(F):
                while nxt < len(todo) and len(pending) < 2 * threads:
                    pending.append((todo[nxt], pool.submit(_decode, paths[todo[nxt]])))
                    nxt += 1
                if unread[i]:
                    flush()
                    continue
                j, fut = pending.popleft()
                t0 = time.perf_counter()
                img, dt = fut.result()
                wait += time.perf_counter() - t0
                decode += dt
                if img is None or img.size == 0:
                    unread[i] = True
                    flush()
                    continue
                if batch and batch_bytes + img.nbytes > memory_budget // 2:
                    flush()
                batch.append((i, img))
                batch_bytes += img.nbytes
            flush()
            _lib.check(L.psfm_colors_result(h, rgb.ctypes.data_as(u8p), C.byref(s)), "psfm_colors_result")
        finally:
            L.psfm_colors_destroy(h)
    rep.unread = [image_names[i] for i in range(F) if unread[i]]
    rep.images = F - len(rep.unread)
    if verbose:
        for i in range(F):
            if unread[i]:
                print(f"Could not read image {image_names[i]} at path {paths[i]}.")
    rep.seconds.update(setup=1e-3 * s.setup_ms, decode=decode, decode_wait=wait, stage=1e-3 * s.stage_ms,
                       upload=1e-3 * s.upload_ms, sample=1e-3 * s.sample_ms, mean=1e-3 * s.mean_ms,
                       total=time.perf_counter() - t_start)
    return rgb, rep


def extract_model_colors(rec, image_path, **kw):
    """Colours every point of the Reconstruction rec in place from its images (all of them: a model read from disk has
    every image registered).  Returns the ColorsReport."""
    ims = list(rec.images.values())
    pts = list(rec.points3D.values())
    sizes = [0 if im.xys is None else len(im.xys) for im in ims]
    kp = [np.asarray(im.xys, np.float64).reshape(-1, 2) for im in ims if im.xys is not None]
    p3 = [np.asarray(im.point3D_ids, np.int64) for im in ims if im.xys is not None]
    rows = point_rows(np.concatenate(p3) if p3 else np.zeros(0, np.int64), [p.point3D_id for p in pts])
    rgb, rep = extract_colors_for_all_images(image_path, [im.name for im in ims],
                                             np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64),
                                             np.concatenate(kp) if kp else np.zeros((0, 2)), rows, len(pts), **kw)
    for p, c in zip(pts, rgb):
        p.rgb = c
    return rep


def main(argv=None):
    ap = argparse.ArgumentParser(prog="color_extractor", description="COLMAP's color_extractor on a binary model")
    ap.add_argument("--image_path", required=True)
    ap.add_argument("--input_path", required=True, help="directory of cameras.bin, images.bin, points3D.bin")
    ap.add_argument("--output_path", required=True)
    args = ap.parse_args(argv)
    rec = colmap_io.read_model(args.input_path)
    extract_model_colors(rec, args.image_path)
    colmap_io.write_model(rec, args.output_path)
    return 0


if __name__ == "__main__":
    sys.exit(main())
