"""python tools/bench_convert.py [--shapes sintel,davis] [--repeats 3] [--out DIR]

Wall time (min, median, max of `repeats` calls, after one warm-up call) of convert.write_depth_pose_from_colmap_format
(the model -> depths/, poses/, intrinsics/ on the device) on synthetic binary models:

    sintel   50 images of 1024 x 436, 12,000 keypoints each (DESIGN §4.9's 600,000 observations over 50 frames)
    davis    80 images of 854 x 480, 20,000 keypoints each (§4.9's 1,600,000 observations over 80 frames)

60 % of the keypoints have a 3D point.  The device call is split into model read, host preparation, upload, counting
pass, kernels and device-to-pinned copies (CUDA events, summed over batches; a batch's copy overlaps the next batch's
kernels), result (wall time of the calls that return the maps) and the .npy / .png / .txt writes (seconds summed over
the writer threads, which run beside the device calls).  The reference arm is oracle/convert_oracle.py's restatement
of sfm/convert.py: the same model read, its loop over every keypoint, np.percentile and the colormap restated in
numpy, this package's PNG encoder in place of plt.imsave, np.save and np.savetxt.  The loop runs over the whole model
in one call of depth_maps_loop, so its point-id lookup table is built once per model, as the reference's points3D dict
is; the display images and files then follow one image at a time, as the reference runs.  It is a restatement, not the
reference itself (matplotlib is not used).  The device name and power limit are
read in the same process.
"""
import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {"sintel": (50, 1024, 436, 12_000), "davis": (80, 854, 480, 20_000)}


def _device_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def make_model(F, W, H, K, seed=0):
    rng = np.random.default_rng(seed)
    P = F * K // 3
    xyz = rng.uniform([-3, -1.5, 2], [3, 1.5, 12], size=(P, 3))
    kps = rng.uniform([0, 0], [W - 1, H - 1], size=(F * K, 2))
    p3 = np.where(rng.random(F * K) < 0.6, rng.integers(0, P, F * K) + 1, -1)
    q = np.column_stack([np.ones(F), rng.normal(0, 0.02, (F, 3))])
    return dict(camera_ids=np.array([1]), camera_size=np.array([[W, H]]), cam_params=np.array([[900.0, W / 2, H / 2]]),
                image_ids=np.arange(1, F + 1), image_names=["%05d.png" % i for i in range(F)],
                image_camera=np.zeros(F, np.int64), qvec=q, tvec=rng.normal(0, 0.1, (F, 3)),
                keypoint_ptr=np.arange(F + 1) * K, keypoints=kps, point3D_ids=p3, point_ids=np.arange(1, P + 1), xyz=xyz,
                error=np.zeros(P), track_ptr=np.zeros(P + 1, np.int64), track_image_ids=np.zeros(0, np.int32),
                track_point2D=np.zeros(0, np.int32))


def reference_arm(model_dir, out):
    """The restated sfm/convert.py: read, the keypoint loop over every image, then per image the display image and
    the files.  Returns the seconds of the read, of the loop and of the whole arm."""
    from oracle import convert_oracle as co
    from particlesfm_b200 import colmap_io, convert
    t0 = time.perf_counter()
    a = convert._model_arrays(colmap_io.read_model(model_dir))
    t_read = time.perf_counter() - t0
    lut = co.binary_lut()
    for d in ("depths", "poses", "intrinsics"):
        os.makedirs(os.path.join(out, d), exist_ok=True)
    t1 = time.perf_counter()
    depths = co.depth_maps_loop(a)
    t_loop = time.perf_counter() - t1
    for i, name in enumerate(a["image_names"]):
        depth = depths[i]
        stem = os.path.splitext(name)[0]
        np.save(os.path.join(out, "depths", stem + ".npy"), depth)
        convert.write_png_rgba(os.path.join(out, "depths", stem + ".png"), co.display_rgba(depth, lut))
        f, cx, cy = a["cam_params"][a["image_camera"][i]][:3]
        np.savetxt(os.path.join(out, "intrinsics", stem + ".txt"), np.array([[f, 0, cx], [0, f, cy], [0, 0, 1]]))
        R = co.qvec2rotmat(a["qvec"][i])
        np.savetxt(os.path.join(out, "poses", stem + ".txt"), np.concatenate([R, a["tvec"][i][:, None]], -1))
    return t_read, t_loop, time.perf_counter() - t0


def _stats(xs):
    return [round(min(xs), 4), round(statistics.median(xs), 4), round(max(xs), 4)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="sintel,davis")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    args = ap.parse_args()
    from particlesfm_b200 import colmap_io, convert, device_count
    if device_count() <= 0:
        raise SystemExit("bench_convert: no CUDA device (the conversion has no CPU path)")
    results = {"device": _device_info(), "shapes": {}}
    for shape in args.shapes.split(","):
        F, W, H, K = SHAPES[shape]
        with tempfile.TemporaryDirectory() as tmp:
            a = make_model(F, W, H, K)
            mdir = os.path.join(tmp, "model")
            colmap_io.write_model_arrays(mdir, *[a[k] for k in (
                "camera_ids", "camera_size", "cam_params", "image_ids", "image_names", "image_camera", "qvec", "tvec",
                "keypoint_ptr", "keypoints", "point3D_ids", "point_ids", "xyz", "error", "track_ptr", "track_image_ids",
                "track_point2D")])
            dev = []
            for r in range(args.repeats + 1):
                out = os.path.join(tmp, "dev%d" % r)
                t0 = time.perf_counter()
                rep = convert.write_depth_pose_from_colmap_format(mdir, out)
                wall = time.perf_counter() - t0
                if r:
                    dev.append(dict(rep.seconds, wall=wall, batches=rep.num_batches))
                shutil.rmtree(out)
            ref = []
            for r in range(args.repeats):
                out = os.path.join(tmp, "ref%d" % r)
                t_read, t_loop, wall = reference_arm(mdir, out)
                ref.append(dict(read=t_read, keypoint_loop=t_loop, wall=wall))
                shutil.rmtree(out)
        row = {"images": F, "size": [W, H], "keypoints_per_image": K, "batches": dev[0]["batches"],
               "device_s": {k: _stats([d[k] for d in dev]) for k in dev[0] if k != "batches"},
               "restated_reference_s": {k: _stats([d[k] for d in ref]) for k in ref[0]}}
        results["shapes"][shape] = row
        print(json.dumps({shape: row}), flush=True)
    print(json.dumps({"device": results["device"]}), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_convert.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
