"""The reconstructed model -> sparse depth maps, display images, poses and intrinsics, on the GPU (DESIGN.md §4.10).

    python -m particlesfm_b200.convert --input_dir MODEL --output_dir OUT

`write_depth_pose_from_colmap_format` has the signature and output of the reference's (sfm/convert.py:43-104).  For
every image of the model, in images.bin order, it writes under OUT:
    depths/NAME.npy       the sparse H x W float64 depth map: z of every keypoint with a 3D point at its rounded,
                          clipped pixel, the last keypoint in keypoint order winning a shared pixel, 0 elsewhere
    depths/NAME.png       its display image: 1 / (depth + 1) between its 2nd and 98th percentiles over the valid
                          (depth > 0) pixels, through matplotlib's `binary` colormap, RGBA8
    poses/NAME.txt        the world-to-camera [R t], R = qvec2rotmat(qvec) as the reference computes it
    intrinsics/NAME.txt   K = [[f, 0, cx], [0, f, cy], [0, 0, 1]] (SIMPLE_PINHOLE, SIMPLE_RADIAL; the distortion term
                          is not used)
NAME is the image name without its extension.  Depth maps and display images come from csrc/convert.cu; the text
files are np.savetxt of the same numpy expressions the reference evaluates, so they are byte-identical to its files.
The PNG is written by a zlib encoder here, so its bytes differ from matplotlib's file; its pixels do not.

Differences from the reference, all refusals before anything is written: an image with no valid pixel is an
IndexError naming it (the reference dies there, leaving the earlier images' files); a text model, an image name with a
path separator and a keypoint whose point3D_id is not in the model (the reference's KeyError) are refused up front.
When two images share an output name, the files of the later one are written, as the reference leaves them.
"""
import argparse
import concurrent.futures
import ctypes as C
import os
import struct
import sys
import time
import zlib

import numpy as np

from . import _abi, _lib, colmap_io

SUPPORTED_MODELS = {0: "SIMPLE_PINHOLE", 2: "SIMPLE_RADIAL"}
DEVICE_BUDGET = 256 << 20          # bytes of device memory for the two batch slots
HOST_BUDGET = 1 << 30              # bytes of maps (12 per pixel) held on the host while they are written


def binary_lut():
    """Bytes of matplotlib's `binary` colormap as plt.imsave writes them: the 256-entry table of
    LinearSegmentedColormap's _create_lookup_table for red = green = blue = ((0, 1, 1), (1, 0, 0)), gamma 1, then
    (value * 255).astype(uint8)."""
    N = 256
    x = np.array([0.0, 1.0]) * (N - 1)
    y0, y1 = np.array([1.0, 0.0]), np.array([1.0, 0.0])
    xind = (N - 1) * np.linspace(0, 1, N) ** 1.0
    ind = np.searchsorted(x, xind)[1:-1]
    distance = (xind[1:-1] - x[ind - 1]) / (x[ind] - x[ind - 1])
    lut = np.clip(np.concatenate([[y1[0]], distance * (y0[ind] - y1[ind - 1]) + y1[ind - 1], [y0[-1]]]), 0.0, 1.0)
    return (lut * 255).astype(np.uint8)


def qvec2rotmat(qvec):
    """The reference's expression (sfm/colmap_utils/read_write_model.py:459-469), term for term."""
    return np.array([
        [1 - 2 * qvec[2]**2 - 2 * qvec[3]**2,
         2 * qvec[1] * qvec[2] - 2 * qvec[0] * qvec[3],
         2 * qvec[3] * qvec[1] + 2 * qvec[0] * qvec[2]],
        [2 * qvec[1] * qvec[2] + 2 * qvec[0] * qvec[3],
         1 - 2 * qvec[1]**2 - 2 * qvec[3]**2,
         2 * qvec[2] * qvec[3] - 2 * qvec[0] * qvec[1]],
        [2 * qvec[3] * qvec[1] - 2 * qvec[0] * qvec[2],
         2 * qvec[2] * qvec[3] + 2 * qvec[0] * qvec[1],
         1 - 2 * qvec[1]**2 - 2 * qvec[2]**2]])


def write_png_rgba(path, rgba, level=6):
    """RGBA8 PNG of rgba [h][w][4] uint8: one IDAT, filter 0 on every row."""
    h, w = rgba.shape[:2]
    raw = np.zeros((h, 1 + 4 * w), np.uint8)
    raw[:, 1:] = rgba.reshape(h, 4 * w)

    def chunk(tag, data):
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xffffffff)

    with open(path, "wb") as f:
        f.write(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 6, 0, 0, 0))
                + chunk(b"IDAT", zlib.compress(raw.tobytes(), level)) + chunk(b"IEND", b""))


class ConvertReport:
    """images (converted), written (images whose files were written: the last of each output name), valid_count [F],
    num_batches, seconds {stage: s} with stages prepare, upload, count, kernels, d2h (CUDA-event times; kernels and d2h
    of consecutive batches overlap), alloc (host wall time of the device and pinned allocations), host_copy (the copies
    from the pinned buffers to the returned maps), result (wall time of the device calls that return the maps, which
    holds kernels, d2h, the slots' alloc and host_copy), npy / png / txt
    (file-writing seconds summed over the writer threads), write_wait (wall time spent waiting for the writers after
    the last maps arrived) and total."""

    def __init__(self):
        self.images, self.written, self.valid_count, self.num_batches, self.seconds = 0, 0, None, 0, {}


def _model_arrays(rec):
    """The flat arrays save_depth_pose_arrays takes, from a Reconstruction (images and points in dict order)."""
    cams = list(rec.cameras.values())
    index = {c.camera_id: j for j, c in enumerate(cams)}
    ims = list(rec.images.values())
    sizes = [0 if im.xys is None else len(im.xys) for im in ims]
    kp = [np.asarray(im.xys, np.float64).reshape(-1, 2) for im in ims if im.xys is not None]
    p3 = [np.asarray(im.point3D_ids, np.int64) for im in ims if im.xys is not None]
    pts = list(rec.points3D.values())
    width = max([len(c.params) for c in cams] + [3])
    params = np.zeros((len(cams), width))
    for j, c in enumerate(cams):
        params[j, :len(c.params)] = c.params
    return dict(camera_ids=np.array([c.camera_id for c in cams], np.int64),
                camera_size=np.array([[c.width, c.height] for c in cams], np.int64).reshape(-1, 2),
                cam_params=params, image_ids=np.array([im.image_id for im in ims], np.int64),
                image_names=[im.name for im in ims],
                image_camera=np.array([index[im.camera_id] for im in ims], np.int64),
                qvec=np.array([im.qvec for im in ims], np.float64).reshape(-1, 4),
                tvec=np.array([im.tvec for im in ims], np.float64).reshape(-1, 3),
                keypoint_ptr=np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64),
                keypoints=np.concatenate(kp) if kp else np.zeros((0, 2)),
                point3D_ids=np.concatenate(p3) if p3 else np.zeros(0, np.int64),
                point_ids=np.array([p.point3D_id for p in pts], np.int64),
                xyz=np.array([p.xyz for p in pts], np.float64).reshape(-1, 3),
                camera_model=np.array([c.model_id for c in cams], np.int64))


def find_model(input_dir):
    """read_model's lookup: INPUT/{cameras,images,points3D}.bin, else INPUT/model/.  A text model is refused."""
    def has(path, ext):
        return all(os.path.isfile(os.path.join(path, n + ext)) for n in ("cameras", "images", "points3D"))
    for path in (input_dir, os.path.join(input_dir, "model")):
        if has(path, ".bin"):
            return path
        if has(path, ".txt"):
            raise ValueError(f"{path} holds a text COLMAP model; only binary models are read (convert it with "
                             "`colmap model_converter --output_type BIN`)")
    raise FileNotFoundError(f"Could not find binary or text COLMAP model at {input_dir}")


def write_depth_pose_from_colmap_format(input_dir, output_dir, memory_budget=DEVICE_BUDGET, host_budget=HOST_BUDGET):
    """sfm/convert.py's entry: the model at input_dir (or input_dir/model) -> depths/, poses/, intrinsics/ under
    output_dir.  Returns a ConvertReport; its seconds gain `read`, the time to read the model."""
    t0 = time.perf_counter()
    rec = colmap_io.read_model(find_model(input_dir))
    read = time.perf_counter() - t0
    rep = save_depth_pose_arrays(output_dir, **_model_arrays(rec), memory_budget=memory_budget, host_budget=host_budget)
    rep.seconds["read"] = read
    rep.seconds["total"] += read
    return rep


def save_depth_pose_arrays(output_dir, camera_ids, camera_size, cam_params, image_ids, image_names, image_camera, qvec,
                           tvec, keypoint_ptr, keypoints, point3D_ids, point_ids, xyz, error=None, track_ptr=None,
                           track_image_ids=None, track_point2D=None, camera_model=0, memory_budget=DEVICE_BUDGET,
                           host_budget=HOST_BUDGET):
    """save_depth_pose on the arrays colmap_io.write_model_arrays takes (the track arrays and errors are not used).
    camera_model: one COLMAP model id for every camera, or one per camera."""
    t_start = time.perf_counter()
    rep = ConvertReport()
    F = len(image_ids)
    camera_size = np.asarray(camera_size, np.int64).reshape(-1, 2)
    nc = len(camera_size)
    cam_params = np.asarray(cam_params, np.float64).reshape(nc, -1)
    models = np.broadcast_to(np.asarray(camera_model, np.int64), (nc,))
    image_camera = np.asarray(image_camera, np.int64)
    qvec, tvec = np.asarray(qvec, np.float64).reshape(-1, 4), np.asarray(tvec, np.float64).reshape(-1, 3)
    kp_ptr = np.asarray(keypoint_ptr, np.int64)
    # host checks, before any launch
    for name in image_names:
        if "/" in name or os.sep in name or (os.altsep and os.altsep in name):
            raise ValueError(f"image name {name!r} contains a path separator")
    if F and (image_camera.min() < 0 or image_camera.max() >= nc):
        raise ValueError("an image's camera index is out of range (camera index)")
    for m in np.unique(models[image_camera]) if F else []:
        if int(m) not in SUPPORTED_MODELS:
            raise NotImplementedError(f"camera model {colmap_io.MODEL_NAMES.get(int(m), int(m))} (only SIMPLE_PINHOLE and "
                                      "SIMPLE_RADIAL)")
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
    xyz = np.ascontiguousarray(np.asarray(xyz, np.float64).reshape(-1, 3))
    keypoints = np.ascontiguousarray(np.asarray(keypoints, np.float64).reshape(-1, 2))
    size32 = np.ascontiguousarray(camera_size, np.int32)
    cam32 = np.ascontiguousarray(image_camera, np.int32)
    lut = np.ascontiguousarray(binary_lut())
    valid = np.zeros(F, np.int64)
    batch_ptr = np.zeros(F + 1, np.int32)
    L = _lib.lib()
    h = C.c_void_p()
    s = _abi.ConvertSummary()
    i64p, ip, u8p = C.POINTER(C.c_int64), C.POINTER(C.c_int32), C.POINTER(C.c_uint8)
    rep.seconds["prepare"] = time.perf_counter() - t_start
    _lib.check(L.psfm_convert_create(nc, size32.ctypes.data_as(ip), F, _lib.dptr(qvec), _lib.dptr(tvec),
                                     cam32.ctypes.data_as(ip), kp_ptr.ctypes.data_as(i64p), _lib.dptr(keypoints),
                                     row.ctypes.data_as(ip), len(xyz), _lib.dptr(xyz), lut.ctypes.data_as(u8p),
                                     int(memory_budget), C.byref(h), valid.ctypes.data_as(i64p),
                                     batch_ptr.ctypes.data_as(ip), C.byref(s)), "psfm_convert_create")
    try:
        rep.images, rep.valid_count, rep.num_batches = F, valid, s.num_batches
        rep.seconds.update(upload=1e-3 * s.upload_ms, count=1e-3 * s.kernel_ms, alloc=1e-3 * s.alloc_ms, kernels=0.0,
                           d2h=0.0, host_copy=0.0, result=0.0, npy=0.0, png=0.0, txt=0.0)
        empty = np.nonzero(valid == 0)[0]
        if len(empty):
            raise IndexError(f"image {image_names[empty[0]]!r} has no pixel with a positive depth: its display "
                             "percentiles do not exist (nothing was written)")
        out = {}
        for d in ("depths", "poses", "intrinsics"):
            out[d] = os.path.join(output_dir, d)
            os.makedirs(out[d], exist_ok=True)
        stem = [os.path.splitext(n)[0] for n in image_names]
        last = {n: i for i, n in enumerate(stem)}
        px = camera_size[image_camera, 0] * camera_size[image_camera, 1]
        px_ptr = np.concatenate([[0], np.cumsum(px)])
        busy = {"npy": 0.0, "png": 0.0, "txt": 0.0}

        def write(i, depth, rgba):
            hh, ww = int(camera_size[image_camera[i], 1]), int(camera_size[image_camera[i], 0])
            t0 = time.perf_counter()
            np.save(os.path.join(out["depths"], stem[i] + ".npy"), depth.reshape(hh, ww))
            t1 = time.perf_counter()
            write_png_rgba(os.path.join(out["depths"], stem[i] + ".png"), rgba.reshape(hh, ww, 4))
            t2 = time.perf_counter()
            f, cx, cy = cam_params[image_camera[i], :3]
            K = np.array([[f, 0, cx], [0, f, cy], [0, 0, 1]])
            np.savetxt(os.path.join(out["intrinsics"], stem[i] + ".txt"), K)
            R, t = qvec2rotmat(qvec[i]), np.expand_dims(tvec[i], -1)
            np.savetxt(os.path.join(out["poses"], stem[i] + ".txt"), np.concatenate([R, t], -1))
            return t1 - t0, t2 - t1, time.perf_counter() - t2

        nb = s.num_batches
        with concurrent.futures.ThreadPoolExecutor(min(32, os.cpu_count() or 1)) as pool:
            pending = []
            j = 0
            while j < nb:
                # a chunk of whole batches inside the host budget, at least one batch
                k = j + 1
                while k < nb and 12 * (px_ptr[batch_ptr[k + 1]] - px_ptr[batch_ptr[j]]) <= host_budget:
                    k += 1
                a, b = int(batch_ptr[j]), int(batch_ptr[k])
                n = int(px_ptr[b] - px_ptr[a])
                depth, rgba = np.empty(n, np.float64), np.empty(4 * n, np.uint8)
                t0 = time.perf_counter()
                _lib.check(L.psfm_convert_result(h, j, k - j, _lib.dptr(depth), rgba.ctypes.data_as(u8p), C.byref(s)),
                           "psfm_convert_result")
                rep.seconds["result"] += time.perf_counter() - t0
                rep.seconds["kernels"] += 1e-3 * s.kernel_ms
                rep.seconds["d2h"] += 1e-3 * s.d2h_ms
                rep.seconds["alloc"] += 1e-3 * s.alloc_ms
                rep.seconds["host_copy"] += 1e-3 * s.host_copy_ms
                for f in pending:                # at most two chunks of maps on the host
                    for key, dt in zip(("npy", "png", "txt"), f.result()):
                        busy[key] += dt
                pending = []
                for i in range(a, b):
                    if last[stem[i]] == i:
                        o = int(px_ptr[i] - px_ptr[a])
                        pending.append(pool.submit(write, i, depth[o:o + px[i]], rgba[4 * o:4 * (o + px[i])]))
                j = k
            t0 = time.perf_counter()
            for f in pending:
                for key, dt in zip(("npy", "png", "txt"), f.result()):
                    busy[key] += dt
            rep.seconds["write_wait"] = time.perf_counter() - t0
        rep.written = len(last)
        rep.seconds.update(busy)
    finally:
        L.psfm_convert_destroy(h)
    rep.seconds["total"] = time.perf_counter() - t_start
    return rep


def main(argv=None):
    ap = argparse.ArgumentParser(description="Read and write COLMAP binary and text models")
    ap.add_argument("--input_dir", help="path to input model folder")
    ap.add_argument("--output_dir", help="path to output model folder")
    args = ap.parse_args(argv)
    rec = colmap_io.read_model(find_model(args.input_dir))
    print("num_cameras:", len(rec.cameras))
    print("num_images:", len(rec.images))
    print("num_points3D:", len(rec.points3D))
    if args.output_dir is not None:
        print(args.output_dir)
        save_depth_pose_arrays(args.output_dir, **_model_arrays(rec))
    return 0


if __name__ == "__main__":
    sys.exit(main())
