"""ParticleSfM's SfM step on the GPU, from the track set and the frames to the converted poses (DESIGN.md §4.12).

    python -m particlesfm_b200.sfm --image_dir I --output_dir O [--traj_dir T] [--assume_static]
                                   [--skip_geometric_verification] [--min_num_matches N] [--quiet]

`main_global_sfm` does what sfm/main_sfm.py:127-159 does and `sfm_reconstruction` what run_particlesfm.py:73-93 does
for `global_theia`, without COLMAP and without a subprocess:

    import        the frames' headers (what `colmap feature_importer` would write, restated below), the track set,
                  then the track set -> ordered matches on the device (handoff, psfm_matches_create) and
                  SFM/image_match_pairs.txt
    table         the database match table on the device (psfm_matches_table) and its host copy for the database
    verification  the geometric verification of the resident table (psfm_match_table_verify), or with
                  skip_geometric_verification the raw matches as config 2 with F = E = H = I
    (mapper)      global_mapper.global_mapper_from_cache on the verification's arrays, coloured from the frames:
                  SFM/model/0/{cameras,images,points3D}.bin, copied to SFM/model/ as compute_model_stats does
    database      the wait for the writer thread, which writes SFM/database.db beside the device work

The database holds what the reference's build_database leaves: the same schema, the cameras and images rows of
feature_importer, the keypoints and matches of import_keypoints_matches and the two-view geometries of
matches_importer.  The mapper reads none of it back.
"""
import argparse
import os
import queue
import shutil
import sqlite3
import sys
import threading
import time

import numpy as np

from . import _lib, convert, global_mapper as gm, handoff, init_geometry

# ---------------------------------------------------------------------------------------------------------------------
# What `colmap feature_importer --ImageReader.single_camera 1 --ImageReader.camera_model SIMPLE_PINHOLE` writes, as
# COLMAP's ImageReader behaves (recalled, not pinned to a source line): every entry of the image directory, sorted by
# name, is one image with image_id 1..N; one SIMPLE_PINHOLE camera, camera_id 1, of the first image's size with
# f = default_focal_length_factor * max(width, height), cx = width / 2, cy = height / 2 and no prior focal length; the
# prior pose columns hold COLMAP's NaN priors, which SQLite stores as NULL.
# ---------------------------------------------------------------------------------------------------------------------
SIMPLE_PINHOLE = 0
CAMERA_ID = 1
DEFAULT_FOCAL_LENGTH_FACTOR = 1.2
EXIF_FOCAL_TAGS = {0x920A: "FocalLength", 0xA405: "FocalLengthIn35mmFilm"}
EXIF_IFD = 0x8769

# the schema of the reference's create_empty_db (sfm/colmap_utils/database.py)
SCHEMA = """
CREATE TABLE IF NOT EXISTS cameras (camera_id INTEGER PRIMARY KEY AUTOINCREMENT NOT NULL, model INTEGER NOT NULL,
    width INTEGER NOT NULL, height INTEGER NOT NULL, params BLOB, prior_focal_length INTEGER NOT NULL);
CREATE TABLE IF NOT EXISTS images (image_id INTEGER PRIMARY KEY AUTOINCREMENT NOT NULL, name TEXT NOT NULL UNIQUE,
    camera_id INTEGER NOT NULL, prior_qw REAL, prior_qx REAL, prior_qy REAL, prior_qz REAL, prior_tx REAL,
    prior_ty REAL, prior_tz REAL, CONSTRAINT image_id_check CHECK(image_id >= 0 and image_id < 2147483647),
    FOREIGN KEY(camera_id) REFERENCES cameras(camera_id));
CREATE TABLE IF NOT EXISTS keypoints (image_id INTEGER PRIMARY KEY NOT NULL, rows INTEGER NOT NULL,
    cols INTEGER NOT NULL, data BLOB, FOREIGN KEY(image_id) REFERENCES images(image_id) ON DELETE CASCADE);
CREATE TABLE IF NOT EXISTS descriptors (image_id INTEGER PRIMARY KEY NOT NULL, rows INTEGER NOT NULL,
    cols INTEGER NOT NULL, data BLOB, FOREIGN KEY(image_id) REFERENCES images(image_id) ON DELETE CASCADE);
CREATE TABLE IF NOT EXISTS matches (pair_id INTEGER PRIMARY KEY NOT NULL, rows INTEGER NOT NULL,
    cols INTEGER NOT NULL, data BLOB);
CREATE TABLE IF NOT EXISTS two_view_geometries (pair_id INTEGER PRIMARY KEY NOT NULL, rows INTEGER NOT NULL,
    cols INTEGER NOT NULL, data BLOB, config INTEGER NOT NULL, F BLOB, E BLOB, H BLOB);
CREATE UNIQUE INDEX IF NOT EXISTS index_name ON images(name);
"""


class ImageSet:
    """The images feature_importer would import: names [N] sorted, image_ids [N] (1..N), the camera's width, height
    and params (f, cx, cy)."""

    def __init__(self, names, width, height):
        self.names = names
        self.image_ids = np.arange(1, len(names) + 1, dtype=np.int64)
        self.width, self.height = width, height
        f = DEFAULT_FOCAL_LENGTH_FACTOR * max(width, height)
        self.camera = np.array([f, width / 2.0, height / 2.0], np.float64)


def read_image_set(image_dir):
    """The ImageSet of image_dir from the images' headers (Pillow, no decoding).  Raises ValueError naming the entry
    for a subdirectory, a file Pillow cannot identify, an image of another size than the first, an image with an EXIF
    focal length (feature_importer would give the camera a prior focal length, and the verification of a pair of such
    cameras, EstimateCalibrated, is not supported), and an empty directory."""
    from PIL import Image, UnidentifiedImageError
    names = sorted(os.listdir(image_dir))
    if not names:
        raise ValueError(f"no images found in {image_dir}")
    size = None
    for name in names:
        path = os.path.join(image_dir, name)
        if os.path.isdir(path):
            raise ValueError(f"{path} is a directory; the image directory must hold image files only")
        try:
            with Image.open(path) as im:
                s = im.size
                exif = im.getexif()
                tags = dict(exif)
                tags.update(exif.get_ifd(EXIF_IFD))
        except (UnidentifiedImageError, OSError) as e:
            raise ValueError(f"{path} is not an image Pillow can identify ({e})") from None
        focal = [EXIF_FOCAL_TAGS[t] for t in EXIF_FOCAL_TAGS if t in tags]
        if focal:
            raise ValueError(f"{path} has an EXIF {focal[0]}: a prior focal length is not supported")
        if size is None:
            size = s
        elif s != size:
            raise ValueError(f"{path} is {s[0]} x {s[1]}, the first image is {size[0]} x {size[1]}; every image must "
                             "have the same size")
    return ImageSet(names, int(size[0]), int(size[1]))


def load_trajectories(trajectories):
    """A trajectory directory holding track.npy (a dict, or a pickled object with .as_dict()), or the dict or
    tracker.TrackArrays itself."""
    if isinstance(trajectories, (str, os.PathLike)):
        return np.load(os.path.join(trajectories, "track.npy"), allow_pickle=True).item()
    return trajectories


def write_schema(db, images):
    """The schema and the cameras and images rows of build_database's create_empty_db and import_images."""
    db.executescript(SCHEMA)
    db.execute("INSERT INTO cameras VALUES (?, ?, ?, ?, ?, ?)",
               (CAMERA_ID, SIMPLE_PINHOLE, images.width, images.height, images.camera.tobytes(), 0))
    db.executemany("INSERT INTO images VALUES (?, ?, ?, NULL, NULL, NULL, NULL, NULL, NULL, NULL)",
                   [(int(i), n, CAMERA_ID) for i, n in zip(images.image_ids, images.names)])
    db.commit()


class DatabaseWriter:
    """One thread that owns the SQLite connection and runs the submitted writes in order.  A failed write skips the
    rest; join() ends the thread and returns that exception (or None).  seconds: the thread's time in writes."""

    def __init__(self, path):
        self.error, self.seconds = None, 0.0
        self._q = queue.Queue()
        self._thread = threading.Thread(target=self._run, args=(path,), name="psfm-sfm-database")
        self._thread.start()

    def submit(self, fn, *args):
        self._q.put((fn, args))

    def _run(self, path):
        db = sqlite3.connect(path)
        try:
            while True:
                item = self._q.get()
                if item is None:
                    return
                if self.error is None:
                    t0 = time.perf_counter()
                    try:
                        item[0](db, *item[1])
                    except BaseException as e:          # handed to the calling thread by join()
                        self.error = e
                    self.seconds += time.perf_counter() - t0
        finally:
            db.close()

    def join(self):
        self._q.put(None)
        self._thread.join()
        return self.error


def mapper_options(min_num_matches=None):
    """The GlobalMapper flags of main_sfm.py:139-149: principal point and extra parameters not refined, and
    min_num_matches when given."""
    o = gm.GlobalMapperOptions(ba_refine_principal_point=False, ba_refine_extra_params=False)
    if min_num_matches:
        o.min_num_matches = int(min_num_matches)
    return o


def main_global_sfm(sfm_dir, image_dir, trajectories, single_camera=True, remove_dynamic=True,
                    skip_geometric_verification=False, min_num_matches=None, convert_path=None):
    """sfm/main_sfm.py:127-159 on the GPU: SFM/database.db, SFM/image_match_pairs.txt and SFM/model/0/*.bin (copied to
    SFM/model/), the points coloured from image_dir.  trajectories: a directory holding track.npy, the dict, a
    tracker.TrackArrays, or a finished tracker._ResidentTracker, whose track set goes into the match table on the device
    (no host copy, no frame-range scan) and which is closed once the table is built.  With convert_path, the converted depth maps and poses are written there from the arrays in
    memory.  Returns a global_mapper.MapperReport whose stages add import, table, verification and database, and whose
    stats are the model's stats (None, and success False, when the rotation or position stage fails and no model is
    written).  Raises ValueError before any device call or file write for an input the importer cannot take."""
    if not single_camera:
        raise ValueError("single_camera=False is not supported: every image would get its own camera, and the bundle "
                         "adjustment refines the focal length of one camera only")
    from .tracker import _ResidentTracker
    report = gm.MapperReport()
    t0 = time.perf_counter()
    images = read_image_set(image_dir)
    resident = isinstance(trajectories, _ResidentTracker)
    if resident:
        # its frame ids are below its number of frames, which the caller has checked against the images
        if trajectories.num_frames > len(images.names):
            raise ValueError(f"the tracker has {trajectories.num_frames} frames, {image_dir} holds {len(images.names)} "
                             "images")
    else:
        flat = handoff._flatten(load_trajectories(trajectories), remove_dynamic)
        frames = flat[2]
        if frames.size and (frames.min() < 0 or frames.max() >= len(images.names)):
            k = int(np.nonzero((frames < 0) | (frames >= len(images.names)))[0][0])
            raise ValueError(f"trajectory {flat[0][int(flat[1][k])]!r} has frame id {int(frames[k])}, not below the "
                             f"number of images ({len(images.names)}) in {image_dir}")
    os.makedirs(sfm_dir, exist_ok=True)
    db_path = os.path.join(sfm_dir, "database.db")
    pair_path = os.path.join(sfm_dir, "image_match_pairs.txt")
    for p in (db_path, pair_path):
        if os.path.exists(p):
            os.remove(p)
    writer = DatabaseWriter(db_path)
    writer.submit(write_schema, images)
    table = None
    try:
        if resident:
            table = handoff.ResidentMatchTable.from_tracker(trajectories, images.image_ids)
            trajectories.close()            # the track set has moved into the table
        else:
            table = handoff.ResidentMatchTable(flat, images.image_ids)
            del flat, frames
        table.pairs.write_pair_list(pair_path, images.names)
        report.add("import", t0, {"images": len(images.names), "ordered_pairs": int(len(table.pairs.pair_images))})
        t0 = time.perf_counter()
        tables = table.tables(images.names, images.camera, (images.width, images.height))
        writer.submit(handoff.insert_rows, *tables.rows())
        report.add("table", t0, {"keypoints": table.num_keypoints, "pairs": table.num_pairs,
                                 "matches": table.num_matches})
        t0 = time.perf_counter()
        if skip_geometric_verification:
            g = tables.unverified_two_view_geometries()
            two_view = tables.rows()[1]
        else:
            ver = init_geometry.verify_match_table(table, tables.image_camera, tables.camera_size)
            g = ver.to_two_view_geometries(tables)
            two_view = ver.two_view_rows(tables.pair_ids)
        table.close()
        writer.submit(handoff.insert_rows, (), (), two_view)
        report.add("verification", t0, {"pairs": int(len(g.pair_ids)), "inlier_matches": int(g.inlier_ptr[-1]),
                                        "skipped": bool(skip_geometric_verification)})
        o = mapper_options(min_num_matches)
        model_path = os.path.join(sfm_dir, "model")
        os.makedirs(model_path, exist_ok=True)
        gm.global_mapper_from_cache(g, handoff.pair_rules(g, o.min_num_matches, o.ignore_watermarks), model_path, o,
                                    convert_path, image_dir, report)
    finally:
        if table is not None:
            table.close()
        t0 = time.perf_counter()
        error = writer.join()
        report.add("database", t0, {"writer_seconds": writer.seconds})
    if error is not None:
        raise error
    if report.success:
        for name in ("cameras.bin", "images.bin", "points3D.bin"):          # compute_model_stats, main_sfm.py:91-92
            shutil.copy(os.path.join(report.output, name), model_path)
    return report


def sfm_reconstruction(image_dir, output_dir, trajectories, assume_static=False):
    """run_particlesfm.py:73-93 for sfm_type global_theia: OUT/sfm by main_global_sfm, then
    OUT/colmap_outputs_converted from the model's arrays in memory.  Without a model (a failed rotation or position
    stage) the database is still complete, and the FileNotFoundError the reference's read_model raises on OUT/sfm is
    raised.  Returns main_global_sfm's report."""
    sfm_dir = os.path.join(output_dir, "sfm")
    report = main_global_sfm(sfm_dir, image_dir, trajectories, remove_dynamic=not assume_static,
                             convert_path=os.path.join(output_dir, "colmap_outputs_converted"))
    if not report.success:
        convert.find_model(sfm_dir)
    return report


# ----------------------------------------------------------------------------- command line

def build_parser():
    ap = argparse.ArgumentParser(prog="sfm", description=__doc__.split("\n\n")[0])
    ap.add_argument("-i", "--image_dir", required=True)
    ap.add_argument("-o", "--output_dir", required=True)
    ap.add_argument("--traj_dir", default=None,
                    help="default OUTPUT_DIR/trajectories_labeled, or OUTPUT_DIR/trajectories with --assume_static")
    ap.add_argument("--assume_static", action="store_true", help="keep the samples labelled dynamic")
    ap.add_argument("--skip_geometric_verification", action="store_true")
    ap.add_argument("--min_num_matches", type=int, default=None)
    ap.add_argument("--quiet", action="store_true")
    # the reference's selectors of paths this library does not build: refused before anything is read
    ap.add_argument("--sfm_type", default="global_theia", help="only global_theia is supported")
    ap.add_argument("--single_camera", type=int, default=1, help="only 1 is supported")
    ap.add_argument("--skip_exists", action="store_true", help="not supported")
    return ap


def unsupported(args):
    """The message for a flag that selects a path this library does not build, or None."""
    if args.sfm_type != "global_theia":
        return f"--sfm_type {args.sfm_type} is not supported (only global_theia)"
    if args.single_camera != 1:
        return f"--single_camera {args.single_camera} is not supported (only 1: one camera for every image)"
    if args.skip_exists:
        return "--skip_exists is not supported"
    return None


def main(argv=None):
    args = build_parser().parse_args(sys.argv[1:] if argv is None else list(argv))
    why = unsupported(args)
    if why:
        print("sfm: " + why, file=sys.stderr)
        return 2
    traj_dir = args.traj_dir or os.path.join(args.output_dir, "trajectories" if args.assume_static else
                                             "trajectories_labeled")
    if not args.quiet:
        print("[ParticleSfM] Running global structure-from-motion with Theia........")
    try:
        sfm_dir = os.path.join(args.output_dir, "sfm")
        rep = main_global_sfm(sfm_dir, args.image_dir, traj_dir, remove_dynamic=not args.assume_static,
                              skip_geometric_verification=args.skip_geometric_verification,
                              min_num_matches=args.min_num_matches,
                              convert_path=os.path.join(args.output_dir, "colmap_outputs_converted"))
    except (ValueError, FileNotFoundError) as e:
        print(f"sfm: {e}", file=sys.stderr)
        return 2
    except _lib.PsfmError as e:
        print(f"sfm: {e}", file=sys.stderr)
        return 1
    if not args.quiet:
        for name, s, _ in rep.stages:
            print(f"sfm: {name:22s} {1e3 * s:9.1f} ms")
    if not rep.success:
        print(f"sfm: Could not reconstruct any model! (the {rep.failed_stage} stage failed: {rep.reason})",
              file=sys.stderr)
        try:
            convert.find_model(sfm_dir)
        except FileNotFoundError as e:
            print(f"sfm: {e}", file=sys.stderr)
        return 1
    print(rep.stats)
    return 0


if __name__ == "__main__":
    sys.exit(main())
