"""COLMAP binary model I/O (cameras.bin / images.bin / points3D.bin) for the HP2 boundary.

The pipeline's output format stays what the reference writes and reads through
`sfm/colmap_utils/read_write_model.py` (`read_model` :419-445, `write_model` :447-456) — the
COLMAP sparse-model layout.  This module reads such a model straight into the
`particlesfm_b200.ba.Reconstruction` the bundle adjuster consumes and writes it back,
with bulk `numpy.frombuffer` decoding of the per-image observation lists and per-point
tracks instead of one `struct.unpack` per element.

Layout (little endian), as documented by COLMAP:
  cameras.bin   u64 n | per camera: i32 id, i32 model, u64 width, u64 height, f64 params[k(model)]
  images.bin    u64 n | per image:  i32 id, f64 q[4], f64 t[3], i32 camera_id, name '\\0',
                                    u64 m, m x (f64 x, f64 y, i64 point3D_id)
  points3D.bin  u64 n | per point:  i64 id, f64 xyz[3], u8 rgb[3], f64 error,
                                    u64 l, l x (i32 image_id, i32 point2D_idx)

tests/test_colmap_io.py checks both directions against files written / parsed by the
reference's own module (tests/golden/colmap_model/, tests/golden/make_colmap_golden.py):
reading them gives the generating values, writing the same model reproduces them byte for byte.
"""
import os
import struct

import numpy as np

from .ba import Camera, Image, Point3D, Reconstruction

# number of parameters per COLMAP camera model id
NUM_PARAMS = {0: 3, 1: 4, 2: 4, 3: 5, 4: 8, 5: 8, 6: 12, 7: 5, 8: 4, 9: 5, 10: 12}
MODEL_NAMES = {0: "SIMPLE_PINHOLE", 1: "PINHOLE", 2: "SIMPLE_RADIAL", 3: "RADIAL", 4: "OPENCV", 5: "OPENCV_FISHEYE",
               6: "FULL_OPENCV", 7: "FOV", 8: "SIMPLE_RADIAL_FISHEYE", 9: "RADIAL_FISHEYE", 10: "THIN_PRISM_FISHEYE"}

_P2D = np.dtype([("x", "<f8"), ("y", "<f8"), ("id", "<i8")])
_TRK = np.dtype([("image_id", "<i4"), ("point2D_idx", "<i4")])


def read_cameras_bin(path):
    buf = open(path, "rb").read()
    (n,), o = struct.unpack_from("<Q", buf, 0), 8
    cams = {}
    for _ in range(n):
        cid, model, w, h = struct.unpack_from("<iiQQ", buf, o)
        o += 24
        if model not in NUM_PARAMS:
            raise ValueError(f"cameras.bin: unknown camera model id {model}")
        k = NUM_PARAMS[model]
        cams[cid] = Camera(cid, model, int(w), int(h), np.frombuffer(buf, "<f8", k, o).copy())
        o += 8 * k
    return cams


def read_images_bin(path):
    buf = open(path, "rb").read()
    (n,), o = struct.unpack_from("<Q", buf, 0), 8
    images = {}
    for _ in range(n):
        iid = struct.unpack_from("<i", buf, o)[0]
        qt = np.frombuffer(buf, "<f8", 7, o + 4)
        cam = struct.unpack_from("<i", buf, o + 60)[0]
        o += 64
        e = buf.index(b"\x00", o)
        name = buf[o:e].decode("utf-8")
        o = e + 1
        (m,) = struct.unpack_from("<Q", buf, o)
        o += 8
        p = np.frombuffer(buf, _P2D, m, o)
        o += 24 * m
        images[iid] = Image(iid, qt[:4].copy(), qt[4:].copy(), cam, name,
                            np.stack([p["x"], p["y"]], axis=1) if m else np.zeros((0, 2)), p["id"].astype(np.int64))
    return images


def read_points3D_bin(path):
    buf = open(path, "rb").read()
    (n,), o = struct.unpack_from("<Q", buf, 0), 8
    pts = {}
    for _ in range(n):
        pid = struct.unpack_from("<q", buf, o)[0]
        xyz = np.frombuffer(buf, "<f8", 3, o + 8).copy()
        rgb = np.frombuffer(buf, np.uint8, 3, o + 32).copy()
        err, l = struct.unpack_from("<dQ", buf, o + 35)
        o += 51
        t = np.frombuffer(buf, _TRK, l, o)
        o += 8 * l
        pts[pid] = Point3D(pid, xyz, rgb, err, t["image_id"].astype(np.int32), t["point2D_idx"].astype(np.int32))
    return pts


def read_model(path):
    """cameras.bin + images.bin + points3D.bin in `path` -> Reconstruction."""
    return Reconstruction(read_cameras_bin(os.path.join(path, "cameras.bin")),
                          read_images_bin(os.path.join(path, "images.bin")),
                          read_points3D_bin(os.path.join(path, "points3D.bin")))


def write_cameras_bin(cameras, path):
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(cameras)))
        for c in cameras.values():
            f.write(struct.pack("<iiQQ", c.camera_id, c.model_id, c.width, c.height))
            f.write(np.asarray(c.params, "<f8").tobytes())


def write_images_bin(images, path):
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(images)))
        for im in images.values():
            f.write(struct.pack("<i", im.image_id))
            f.write(np.asarray(im.qvec, "<f8").tobytes())
            f.write(np.asarray(im.tvec, "<f8").tobytes())
            f.write(struct.pack("<i", im.camera_id))
            f.write(im.name.encode("utf-8") + b"\x00")
            m = 0 if im.xys is None else len(im.xys)
            f.write(struct.pack("<Q", m))
            if m:
                p = np.empty(m, _P2D)
                p["x"], p["y"], p["id"] = im.xys[:, 0], im.xys[:, 1], im.point3D_ids
                f.write(p.tobytes())


def write_points3D_bin(points3D, path):
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(points3D)))
        for p in points3D.values():
            f.write(struct.pack("<q", p.point3D_id))
            f.write(np.asarray(p.xyz, "<f8").tobytes())
            f.write(np.asarray(p.rgb if p.rgb is not None else (0, 0, 0), np.uint8).tobytes())
            l = 0 if p.image_ids is None else len(p.image_ids)
            f.write(struct.pack("<dQ", p.error, l))
            if l:
                t = np.empty(l, _TRK)
                t["image_id"], t["point2D_idx"] = p.image_ids, p.point2D_idxs
                f.write(t.tobytes())


def write_model(reconstruction, path):
    os.makedirs(path, exist_ok=True)
    write_cameras_bin(reconstruction.cameras, os.path.join(path, "cameras.bin"))
    write_images_bin(reconstruction.images, os.path.join(path, "images.bin"))
    write_points3D_bin(reconstruction.points3D, os.path.join(path, "points3D.bin"))


_PT_CHUNK = 1 << 16
_PT_HDR = np.dtype([("id", "<i8"), ("xyz", "<f8", 3), ("rgb", "u1", 3), ("error", "<f8"), ("len", "<u8")])   # 51 bytes


def write_model_arrays(path, camera_ids, camera_size, cam_params, image_ids, image_names, image_camera, qvec, tvec,
                       keypoint_ptr, keypoints, point3D_ids, point_ids, xyz, error, track_ptr, track_image_ids,
                       track_point2D, camera_model=0, rgb=None):
    """cameras.bin, images.bin and points3D.bin from flat arrays, byte for byte what write_model writes for the
    equivalent Reconstruction (cameras, images and points in array order).
      cameras   camera_ids [C], camera_size [C][2] (width, height), cam_params [C][k] of `camera_model`
      images    the images to write: image_ids [F], image_names [F], image_camera [F] (index into the cameras),
                qvec [F][4], tvec [F][3], keypoint_ptr [F + 1] over keypoints [K][2] and point3D_ids [K] (-1: none)
      points    point_ids [P], xyz [P][3], error [P], track_ptr [P + 1] over track_image_ids / track_point2D [E],
                rgb [P][3] uint8 (None: every point black)
    The per-observation and per-track-element bytes are laid out with numpy, without a loop over them."""
    os.makedirs(path, exist_ok=True)
    cam_params = np.asarray(cam_params, "<f8").reshape(len(camera_ids), -1)
    with open(os.path.join(path, "cameras.bin"), "wb") as f:
        f.write(struct.pack("<Q", len(camera_ids)))
        for c in range(len(camera_ids)):
            f.write(struct.pack("<iiQQ", int(camera_ids[c]), int(camera_model), int(camera_size[c][0]), int(camera_size[c][1])))
            f.write(cam_params[c].tobytes())
    kp_ptr = np.asarray(keypoint_ptr, np.int64)
    obs = np.empty(kp_ptr[-1], _P2D)
    kps = np.asarray(keypoints).reshape(-1, 2)
    obs["x"], obs["y"], obs["id"] = kps[:, 0], kps[:, 1], point3D_ids
    obs = obs.view(np.uint8).reshape(-1)
    q, t = np.asarray(qvec, "<f8").reshape(-1, 4), np.asarray(tvec, "<f8").reshape(-1, 3)
    with open(os.path.join(path, "images.bin"), "wb") as f:
        f.write(struct.pack("<Q", len(image_ids)))
        cam_ids = np.asarray(camera_ids)[np.asarray(image_camera, np.int64)] if len(image_ids) else []
        for i in range(len(image_ids)):
            lo, hi = int(kp_ptr[i]), int(kp_ptr[i + 1])
            f.write(struct.pack("<i", int(image_ids[i])) + q[i].tobytes() + t[i].tobytes() + struct.pack("<i", int(cam_ids[i]))
                    + image_names[i].encode("utf-8") + b"\x00" + struct.pack("<Q", hi - lo))
            f.write(obs[24 * lo:24 * hi].tobytes())
    P = len(point_ids)
    tp = np.asarray(track_ptr, np.int64)
    xyz = np.asarray(xyz).reshape(-1, 3)
    with open(os.path.join(path, "points3D.bin"), "wb") as f:
        f.write(struct.pack("<Q", P))
        # points in chunks, so that the byte-placement indices stay bounded (8 B per output byte of one chunk: about
        # 27 MB for the chunk's headers plus 64 B per track element) whatever the model's size
        for a in range(0, P, _PT_CHUNK):
            b = min(P, a + _PT_CHUNK)
            lo, hi = int(tp[a]), int(tp[b])
            hdr = np.zeros(b - a, _PT_HDR)
            hdr["id"], hdr["xyz"], hdr["error"], hdr["len"] = point_ids[a:b], xyz[a:b], error[a:b], np.diff(tp[a:b + 1])
            if rgb is not None:
                hdr["rgb"] = np.asarray(rgb, np.uint8).reshape(-1, 3)[a:b]
            trk = np.empty(hi - lo, _TRK)
            trk["image_id"], trk["point2D_idx"] = track_image_ids[lo:hi], track_point2D[lo:hi]
            # within the chunk, point p's header starts at 51 p + 8 (track_ptr[p] - lo); element e at 51 (p + 1) + 8 e
            out = np.empty(51 * (b - a) + 8 * (hi - lo), np.uint8)
            h0 = 51 * np.arange(b - a, dtype=np.int64) + 8 * (tp[a:b] - lo)
            out[(h0[:, None] + np.arange(51)).reshape(-1)] = hdr.view(np.uint8)
            e0 = 51 * (np.repeat(np.arange(b - a, dtype=np.int64), np.diff(tp[a:b + 1])) + 1) + 8 * np.arange(hi - lo, dtype=np.int64)
            out[(e0[:, None] + np.arange(8)).reshape(-1)] = trk.view(np.uint8)
            f.write(out.tobytes())
