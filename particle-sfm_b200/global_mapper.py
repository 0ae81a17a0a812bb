"""gcolmap global_mapper on the GPU: from a verified COLMAP database to a written model (DESIGN.md §4.9).

    python -m particlesfm_b200.global_mapper --database_path DB --output_path OUT [--GlobalMapper.* flags]

GlobalMapperController::Reconstruct (reference controllers/global_mapper.cc:136-184), every stage on the device:

     1  database cache              handoff.load_database_cache (DatabaseCache::Load pair rules); stages 2-14 are
                                    global_mapper_from_cache, which takes the cache from memory
     2  relative poses              init_geometry.estimate_relative_poses, then the cache drops what it leaves UNDEFINED
     3  rotations                   init_geometry.estimate_global_rotations
     4  pairwise translations       init_geometry.optimize_pairwise_translations on the rotation stage's kept pairs
     5  positions (LUD)             init_geometry.estimate_global_positions
     6  registration                tvec = -R c (RegisterAllImages)
     7  triangulation               init_geometry.triangulate_all_points_resident on the cache's pairs
     8  hand-off                    ba.TriangulationSolver (psfm_ba_create_from_triangulation), gauge on the two
                                    smallest registered ids
     9  refinement pass A           psfm_ba_iterative_refinement, known rotations
    10  refinement pass B           the same resident solver, rotations and focal length
    11  model                       psfm_ba_get_model
    12  colors (image_path set and  colors.extract_colors_for_all_images on the registered images: each point's
        extract_colors)             mean bilinear colour (ExtractColorsForAllImages, DESIGN.md §4.11)
    13  write                       colmap_io.write_model_arrays -> OUT/0/{cameras,images,points3D}.bin
    14  convert (convert_path set)  convert.save_depth_pose_arrays on the same arrays -> CONVERT/{depths,poses,
                                    intrinsics}, what sfm/convert.py writes from the model (DESIGN.md §4.10)

The model differs from gcolmap's by exactly the steps this library does not run: CompleteAndMergeTracks and
Retriangulate inside the refinement loop, FilterImages after it, and, without an image path, the colour extraction
(points are then written with rgb 0).  Images that cannot be read leave their observations out of the colours, as in
the reference; they are listed in the colors stage's summary and are not an error.  As in the reference, a failed
rotation or position stage leaves no model and is not an error: the run ends with exit status 0 and no OUT/0.
"""
import argparse
import ctypes as C
import os
import sys
import time

import numpy as np

from . import _abi, _lib, ba, colmap_io, colors, convert, handoff, init_geometry

# the reference steps this mapper leaves out; ExtractColors only when no image path is given (or extract_colors is off)
NOT_RUN = ("CompleteAndMergeTracks", "Retriangulate", "FilterImages", "ExtractColors")


class GlobalMapperOptions:
    """GlobalMapperOptions (controllers/global_mapper.h:32-75) with the reference's names and defaults, the
    GlobalMapper::Options thresholds the refinement loop reads (sfm/global_mapper.h:45-56), and the stage options the
    mapper hands on: rotation (RobustRotationEstimatorOptions), lud (ConstrainedL1SolverOptions), triangulation
    (IncrementalTriangulatorOptions)."""

    def __init__(self, **kw):
        self.min_num_matches = 15
        self.ignore_watermarks = False
        self.num_threads = -1                       # meaningless on the GPU; kept for the surface
        self.extract_colors = True                  # with an image path: the colors stage
        self.min_track_length = 2
        self.max_track_length = 2 ** 31 - 1
        self.min_focal_length_ratio = 0.1
        self.max_focal_length_ratio = 10.0
        self.max_extra_param = 1.0
        self.ba_refine_focal_length = True
        self.ba_refine_principal_point = False
        self.ba_refine_extra_params = True
        self.ba_fix_prior_rotation = False
        self.ba_min_num_residuals_for_multi_threading = 50000
        self.ba_global_max_num_iterations = 50
        self.ba_global_max_refinements = 5
        self.ba_global_max_refinement_change = 0.0005
        self.fix_existing_images = False
        self.camera_path = ""
        self.filter_max_reproj_error = 4.0
        self.filter_min_tri_angle = 1.5
        self.rotation = init_geometry.RobustRotationEstimatorOptions()
        self.lud = init_geometry.ConstrainedL1SolverOptions()
        self.triangulation = init_geometry.IncrementalTriangulatorOptions()
        for k, v in kw.items():
            if not hasattr(self, k):
                raise TypeError(f"GlobalMapperOptions has no option {k!r}")
            setattr(self, k, v)

    def triangulator_options(self):
        """GlobalMapperOptions::Triangulation(): the bogus-camera thresholds come from the mapper's options."""
        t = self.triangulation
        fields = {n: getattr(t, n) for n, _ in _abi.TriangulatorOptions._fields_}
        fields.update(min_focal_length_ratio=self.min_focal_length_ratio, max_focal_length_ratio=self.max_focal_length_ratio,
                      max_extra_param=self.max_extra_param)
        return init_geometry.IncrementalTriangulatorOptions(**fields)


class MapperReport:
    """success (a model was written), failed_stage (None, "rotations" or "positions") and reason (why it failed),
    stages [(name, seconds, summary dict)], output (the model directory or None), not_run (the reference steps this
    mapper does not run), stats (model_stats of the written model, or None)."""

    def __init__(self):
        self.success, self.failed_stage, self.reason, self.output = False, None, None, None
        self.stages, self.not_run = [], NOT_RUN
        self.stats = None

    def add(self, name, t0, summary=None):
        self.stages.append((name, time.perf_counter() - t0, summary or {}))

    def seconds(self, name):
        return sum(s for n, s, _ in self.stages if n == name)


def _refine_options(o, force_update_rotation):
    return ba._global_ba_options(force_update_rotation, o.ba_refine_focal_length, o.ba_refine_principal_point,
                                 o.ba_refine_extra_params, o.ba_fix_prior_rotation, o.ba_global_max_num_iterations, True,
                                 _abi.SOLVER_AUTO).to_struct()


def poses_and_points(g, used, o, report):
    """Stages 2-7 on a cache (g, used): returns (pair_used, rotations, positions, ResidentTriangulation), or None when
    the rotation or position stage fails (report.failed_stage says which)."""
    t0 = time.perf_counter()
    poses = init_geometry.estimate_relative_poses(**g.relative_pose_inputs())
    used = handoff.cache_after_relative_pose(used, poses)
    report.add("relative_poses", t0, {"pairs": int(len(used)), "pairs_used": int(used.sum()),
                                      "estimated": int((poses.estimated & used).sum())})
    F = len(g.image_ids)
    t0 = time.perf_counter()
    rot = init_geometry.estimate_global_rotations(F, g.pair_images, poses.qvec, np.diff(g.inlier_ptr),
                                                  has_pose=poses.estimated & used, options=o.rotation)
    report.add("rotations", t0, dict(rot.summary, success=rot.success, images=int(rot.has_orientation.sum()),
                                     pairs_kept=int(rot.pair_kept.sum())))
    if not rot.success:
        report.failed_stage, report.reason = "rotations", "no posed pair, or the rotation averaging failed"
        return None
    db = {k: getattr(g, k) for k in ("keypoint_ptr", "keypoints", "image_camera", "cameras", "pair_images", "inlier_ptr",
                                     "inlier_matches")}
    t0 = time.perf_counter()
    t = init_geometry.optimize_pairwise_translations(**db, orientations=rot.orientations, pair_used=rot.pair_kept)
    report.add("pairwise_translations", t0, {"pairs": int(rot.pair_kept.sum())})
    t0 = time.perf_counter()
    try:
        pos = init_geometry.estimate_global_positions(F, g.pair_images, t, rot.orientations,
                                                      has_orientation=rot.has_orientation, pair_used=rot.pair_kept,
                                                      options=o.lud)
    except _lib.PsfmError as e:
        # no used pair, a disconnected graph or a failed factorisation (PSFM_ERR_INVALID): EstimatePositions returns
        # false.  Every other status (a device fault, an unsupported size) is an error of this run, not of the scene.
        if e.code != _abi.PSFM_ERR_INVALID:
            raise
        report.add("positions", t0, {"error": str(e)})
        report.failed_stage, report.reason = "positions", str(e)
        return None
    report.add("positions", t0, dict(pos.summary, registered=int(pos.has_position.sum())))
    if pos.has_position.sum() < 2:
        report.failed_stage, report.reason = "positions", "fewer than two images have a position"
        return None
    t0 = time.perf_counter()
    tri = init_geometry.triangulate_all_points_resident(**db, camera_size=g.camera_size, orientations=rot.orientations,
                                                        image_tvec=pos.image_tvec, registered=pos.has_position,
                                                        pair_used=used, options=o.triangulator_options())
    report.add("triangulation", t0, tri.summary)
    return used, rot, pos, tri


def global_mapper(database_path, output_path, options=None, convert_path=None, image_path=None):
    """Run the mapper on `database_path` and write OUT/0/{cameras,images,points3D}.bin under `output_path`.  Returns
    a MapperReport; a failed rotation or position stage writes nothing and is not an exception.  With image_path and
    options.extract_colors, the points are coloured from the registered images under image_path (stage `colors`; its
    summary lists the images that could not be read, which are not an error).  With convert_path,
    the model's depth maps, poses and intrinsics are then written there from the arrays in memory (stage `convert`),
    as convert.write_depth_pose_from_colmap_format would write them from OUT/0.  OUT/0 is written first: a registered
    image with no pixel of positive depth leaves it in place, writes nothing under convert_path and raises the
    conversion's IndexError instead of returning a report."""
    o = options or GlobalMapperOptions()
    report = MapperReport()
    t0 = time.perf_counter()
    g, used = handoff.load_database_cache(database_path, o.min_num_matches, o.ignore_watermarks)
    report.add("database_cache", t0, {"images": int(len(g.image_ids)), "pairs": int(len(used)), "pairs_used": int(used.sum())})
    return global_mapper_from_cache(g, used, output_path, o, convert_path, image_path, report)


def global_mapper_from_cache(g, used, output_path, options=None, convert_path=None, image_path=None, report=None):
    """Stages 2-14 of global_mapper on a database cache already in memory: g a handoff.TwoViewGeometries, used its
    pair_used (handoff.pair_rules).  The stages are appended to `report` (a new MapperReport when None), which is
    returned; everything else is as global_mapper.  A written model's stats are in report.stats (model_stats)."""
    o = options or GlobalMapperOptions()
    report = report if report is not None else MapperReport()
    staged = poses_and_points(g, used, o, report)
    if staged is None:
        return report
    _, rot, pos, tri = staged
    reg = np.nonzero(pos.has_position)[0]
    try:
        t0 = time.perf_counter()
        pose_constant = np.zeros(len(g.image_ids), np.uint8)
        tmask = np.zeros(len(g.image_ids), np.uint8)
        pose_constant[reg[0]] = 1                  # fix 7 DoF (sfm/global_mapper.cc:431-435)
        tmask[reg[1]] = 1
        S = ba.TriangulationSolver(tri, rot.orientations, pos.image_tvec, g.cameras, pose_constant, tmask)
    finally:
        tri.close()
    try:
        report.add("handoff", t0, {"images": S.num_images, "points": S.num_points, "observations": S.num_observations})
        ro = _abi.BARefineOptions()
        _lib.lib().psfm_ba_default_refine_options(C.byref(ro))
        ro.max_refinements = o.ba_global_max_refinements
        ro.max_refinement_change = o.ba_global_max_refinement_change
        ro.filter_max_reproj_error = o.filter_max_reproj_error
        ro.filter_min_tri_angle = o.filter_min_tri_angle
        for name, force in (("refinement_A", False), ("refinement_B", True)):
            t0 = time.perf_counter()
            rep = S.iterative_refinement(_refine_options(o, force), ro)
            report.add(name, t0, {"rounds": rep.num_rounds, "final_num_observations": rep.final_num_observations,
                                  "ba_iterations": list(rep.ba_iterations)[:rep.num_rounds]})
        t0 = time.perf_counter()
        model = S.get_model(len(g.keypoints))
        report.add("model", t0)
    finally:
        S.close()
    arrays = model_arrays(g, pos.has_position, model)
    rgb = None
    if image_path is not None and o.extract_colors:
        t0 = time.perf_counter()
        rgb, c = colors.extract_colors_for_all_images(image_path, arrays[4], arrays[8], arrays[9],
                                                      colors.point_rows(arrays[10], arrays[11]), len(arrays[11]),
                                                      verbose=False)
        report.add("colors", t0, {"images": c.images, "unread": c.unread, "batches": c.num_batches,
                                  "observations": c.num_observations})
        report.not_run = tuple(n for n in NOT_RUN if n != "ExtractColors")
    t0 = time.perf_counter()
    out = os.path.join(output_path, "0")
    colmap_io.write_model_arrays(out, *arrays, rgb=rgb)
    report.add("write", t0, {"points": int((np.diff(model.track_ptr) > 0).sum()), "observations": int(model.track_ptr[-1])})
    report.stats = model_stats(arrays)
    if convert_path is not None:
        t0 = time.perf_counter()
        c = convert.save_depth_pose_arrays(convert_path, *arrays)
        report.add("convert", t0, {"images": c.images, "batches": c.num_batches})
    report.success, report.output = True, out
    return report


def model_stats(arrays):
    """The six numbers sfm/main_sfm.py:73-90 parses from `colmap model_analyzer`, from model_arrays' arrays:
    registered images, points, observations, mean track length, mean observations per registered image, and the mean
    reprojection error as Reconstruction::ComputeMeanReprojectionError computes it (recalled: the mean of the points'
    errors over the points that have one, error != -1; 0 without any).  The means are exact; model_analyzer prints
    them with six decimals."""
    images, point_ids, error, track_ptr = arrays[3], arrays[11], np.asarray(arrays[13], np.float64), arrays[14]
    reg, pts, obs = len(images), len(point_ids), int(track_ptr[-1])
    has = error != -1.0
    return {"num_reg_images": reg, "num_sparse_points": pts, "num_observations": obs,
            "mean_track_length": obs / pts if pts else 0.0, "num_observations_per_image": obs / reg if reg else 0.0,
            "mean_reproj_error": float(error[has].mean()) if has.any() else 0.0}


def write_model(path, g, registered, model):
    """OUT/0 of a TriangulationModel: every camera, the registered images with all their keypoints, the points that
    kept an observation (id = row + 1)."""
    colmap_io.write_model_arrays(path, *model_arrays(g, registered, model))


def model_arrays(g, registered, model):
    """The positional arguments of colmap_io.write_model_arrays after its path, for write_model."""
    reg = np.nonzero(registered)[0]
    sizes = np.diff(g.keypoint_ptr)
    sel = np.repeat(np.asarray(registered, bool), sizes)        # the keypoints of the registered images
    p3 = model.point3D_of_keypoint[sel]
    alive = np.nonzero(np.diff(model.track_ptr) > 0)[0]
    # a deleted point has an empty track, so the elements of the kept points are all of them, in order
    return (
        g.camera_ids, g.camera_size, model.cam_params, g.image_ids[reg], [g.image_names[f] for f in reg],
        g.image_camera[reg], model.qvec[reg], model.tvec[reg], np.concatenate([[0], np.cumsum(sizes[reg])]),
        np.asarray(g.keypoints, np.float64)[sel], np.where(p3 >= 0, p3 + 1, -1), alive + 1, model.xyz[alive],
        model.error[alive], np.concatenate([[0], model.track_ptr[alive + 1]]), np.asarray(g.image_ids)[model.track_image],
        model.track_point2D)


# ----------------------------------------------------------------------------- command line

def _flag(ap, name, default, help_=""):
    ap.add_argument(f"--GlobalMapper.{name}", dest=name, type=type(default) if not isinstance(default, bool) else int,
                    default=int(default) if isinstance(default, bool) else default, help=help_)


def build_parser():
    ap = argparse.ArgumentParser(prog="global_mapper", description=__doc__.split("\n\n")[0])
    ap.add_argument("--database_path", required=True)
    ap.add_argument("--image_path", default="", help="the images, to colour the points (empty: every point black)")
    ap.add_argument("--output_path", required=True, help="the model is written to OUTPUT_PATH/0")
    ap.add_argument("--random_seed", type=int, default=0, help="accepted; every stage is deterministic")
    ap.add_argument("--quiet", action="store_true")
    d = GlobalMapperOptions()
    for name in ("num_threads", "min_num_matches", "ignore_watermarks", "ba_refine_focal_length", "ba_refine_principal_point",
                 "ba_refine_extra_params", "ba_global_max_num_iterations", "ba_global_max_refinements",
                 "ba_global_max_refinement_change", "filter_max_reproj_error", "filter_min_tri_angle"):
        _flag(ap, name, getattr(d, name))
    _flag(ap, "fix_prior_rotation", False, "keep rotations fixed in pass B too")
    _flag(ap, "extract_colors", True, "colour the points from the images under --image_path")
    # the reference's selectors of paths this mapper does not build: refused before any device call
    _flag(ap, "filter_with_1dsfm", False, "only 0 is supported")
    ap.add_argument("--GlobalMapper.position_method", dest="position_method", default="lud", help="only lud is supported")
    _flag(ap, "lud_use_scale_constraints", False, "only 0 is supported")
    return ap


def unsupported(args):
    """The message for a flag that selects a path this mapper does not build, or None."""
    if args.filter_with_1dsfm:
        return "--GlobalMapper.filter_with_1dsfm 1 (the 1DSfM translation filter) is not supported"
    if args.position_method != "lud":
        return f"--GlobalMapper.position_method {args.position_method} is not supported (only lud)"
    if args.lud_use_scale_constraints:
        return "--GlobalMapper.lud_use_scale_constraints 1 is not supported"
    return None


def options_from_args(args):
    keep = ("num_threads", "min_num_matches", "ignore_watermarks", "ba_refine_focal_length", "ba_refine_principal_point",
            "ba_refine_extra_params", "ba_global_max_num_iterations", "ba_global_max_refinements",
            "ba_global_max_refinement_change", "filter_max_reproj_error", "filter_min_tri_angle")
    o = GlobalMapperOptions(**{k: getattr(args, k) for k in keep})
    for k in ("ignore_watermarks", "ba_refine_focal_length", "ba_refine_principal_point", "ba_refine_extra_params"):
        setattr(o, k, bool(getattr(o, k)))
    o.ba_fix_prior_rotation = bool(args.fix_prior_rotation)
    o.extract_colors = bool(args.extract_colors)
    return o


def main(argv=None):
    argv = sys.argv[1:] if argv is None else list(argv)
    if argv[:1] == ["global_mapper"]:          # called as gcolmap is: `<binary> global_mapper --database_path ...`
        argv = argv[1:]
    args = build_parser().parse_args(argv)
    why = unsupported(args)
    if why:
        print("global_mapper: " + why, file=sys.stderr)
        return 2
    if not os.path.exists(args.database_path):
        print(f"global_mapper: no database at {args.database_path}", file=sys.stderr)
        return 2
    try:
        rep = global_mapper(args.database_path, args.output_path, options_from_args(args),
                            image_path=args.image_path or None)
    except _lib.PsfmError as e:
        print(f"global_mapper: {e}", file=sys.stderr)
        return 1
    if not args.quiet:
        for name, s, summary in rep.stages:
            if name == "colors":
                for n in summary["unread"]:
                    print(f"Could not read image {n} at path {os.path.join(args.image_path, n)}.")
            print(f"global_mapper: {name:22s} {1e3 * s:9.1f} ms")
        if rep.success:
            print(f"global_mapper: wrote {rep.output} (not run: {', '.join(rep.not_run)})")
    if not rep.success:       # the reference's outcome too: no model, exit status 0; the reason is always printed
        print(f"global_mapper: => Global {rep.failed_stage[:-1]} failed ({rep.reason}); no model written", file=sys.stderr)
    return 0


if __name__ == "__main__":
    sys.exit(main())
