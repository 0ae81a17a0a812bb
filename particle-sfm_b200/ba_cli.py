"""psfm_ba — global bundle adjustment of a COLMAP model directory on the GPU (HP2, boundary B3).

    python -m particlesfm_b200.ba_cli --input_path M --output_path M' [options]

The process-level surface of the reference is `gcolmap global_mapper --database_path ...
--output_path OUT` (exe/gcolmap.cc:77-85, called from sfm/main_sfm.py:139-152), which cannot be
built here (COLMAP / Theia).  This driver is the slice of it that this library replaces: it reads
`M/{cameras,images,points3D}.bin` (the format gcolmap writes, base/reconstruction.cc:1912-1989),
runs what GlobalMapperController::Run does after triangulation (controllers/global_mapper.cc:177-178)

    IterativeGlobalRefinement(force_update_rotation = false)   # known rotation: translations + points
    IterativeGlobalRefinement(force_update_rotation = true)    # joint, + focal length

on the device (psfm_ba_iterative_refinement: negative-depth filter, BA, Normalize, point filters,
<= 5 rounds each) and writes the model back in the same format, so that it slots between
triangulation and sfm/convert.py.  Option names follow the reference's `--GlobalMapper.*` flags
(controllers/global_mapper.h:46-75, sfm/main_sfm.py:144-150).
"""
import argparse
import sys
import time

from . import _abi, ba, colmap_io


def _flag(ap, name, default, help_):
    ap.add_argument(f"--GlobalMapper.{name}", dest=name, type=type(default) if not isinstance(default, bool) else int,
                    default=int(default) if isinstance(default, bool) else default, help=help_)


def build_parser():
    ap = argparse.ArgumentParser(prog="psfm_ba", description=__doc__.split("\n\n")[0])
    ap.add_argument("--input_path", required=True, help="directory with cameras.bin, images.bin, points3D.bin")
    ap.add_argument("--output_path", required=True)
    _flag(ap, "ba_refine_focal_length", True, "pass B refines the focal length (sfm/main_sfm.py:148)")
    _flag(ap, "ba_refine_principal_point", False, "")
    _flag(ap, "ba_refine_extra_params", False, "")
    _flag(ap, "ba_fix_prior_rotation", False, "keep rotations fixed in pass B too")
    _flag(ap, "ba_global_max_num_iterations", 50, "")
    _flag(ap, "ba_global_max_refinements", 5, "")
    _flag(ap, "ba_global_max_refinement_change", 0.0005, "")
    _flag(ap, "filter_max_reproj_error", 4.0, "")
    _flag(ap, "filter_min_tri_angle", 1.5, "")
    ap.add_argument("--skip_known_rotation_pass", action="store_true", help="run only the joint pass")
    ap.add_argument("--linear_solver", default="auto", choices=["auto", "exact", "iterative"],
                    help="auto = the reference rule: exact Schur for <= 1000 images (bundle_adjustment.cc:276-286)")
    ap.add_argument("--quiet", action="store_true")
    return ap


def run(args):
    solver = {"auto": _abi.SOLVER_AUTO, "exact": _abi.SOLVER_EXACT_SCHUR, "iterative": _abi.SOLVER_ITERATIVE_SCHUR}[args.linear_solver]
    rec = colmap_io.read_model(args.input_path)
    for c in rec.cameras.values():
        if c.model_id != ba.SIMPLE_PINHOLE:
            raise SystemExit(f"psfm_ba: camera {c.camera_id} is {colmap_io.MODEL_NAMES.get(c.model_id, c.model_id)}; the pipeline "
                             "imports features with SIMPLE_PINHOLE (sfm/import_feature_matches.py:50-58) and only that model is supported")
    say = (lambda *a: None) if args.quiet else (lambda *a: print(*a, flush=True))
    say(f"psfm_ba: {len(rec.images)} images, {len(rec.points3D)} points, {rec.ComputeNumObservations()} observations")
    kw = dict(ba_refine_focal_length=bool(args.ba_refine_focal_length),
              ba_refine_principal_point=bool(args.ba_refine_principal_point),
              ba_refine_extra_params=bool(args.ba_refine_extra_params), ba_fix_prior_rotation=bool(args.ba_fix_prior_rotation),
              ba_global_max_num_iterations=args.ba_global_max_num_iterations,
              ba_global_max_refinements=args.ba_global_max_refinements,
              ba_global_max_refinement_change=args.ba_global_max_refinement_change,
              filter_max_reproj_error=args.filter_max_reproj_error, filter_min_tri_angle=args.filter_min_tri_angle,
              quiet=args.quiet, linear_solver=solver)
    reports = []
    for force_update_rotation in ((True,) if args.skip_known_rotation_pass else (False, True)):
        say("=" * 78 + "\n" + ("Global bundle adjustment" if force_update_rotation else "Global bundle adjustment (Known rotation)")
            + "\n" + "=" * 78)
        t0 = time.perf_counter()
        rep = ba.iterative_global_refinement(rec, force_update_rotation, **kw)
        reports.append(rep)
        for k, r in enumerate(rep.rounds()):
            say(f"  round {k + 1}: {r['num_observations']} observations, {r['ba_iterations']} LM iterations, final cost {r['final_cost']:.6g}"
                f"\n  => Filtered observations: {r['changed_observations']}\n  => Changed observations: {r['changed']:.6f}")
        say(f"  {rep.final_num_observations} observations left, {time.perf_counter() - t0:.3f} s")
    colmap_io.write_model(rec, args.output_path)
    say(f"psfm_ba: wrote {args.output_path} ({len(rec.points3D)} points, {rec.ComputeNumObservations()} observations)")
    return reports


def main(argv=None):
    run(build_parser().parse_args(argv))
    return 0


if __name__ == "__main__":
    sys.exit(main())
