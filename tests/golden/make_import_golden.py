"""Generates tests/golden/import_small.npz by running the REFERENCE's import_keypoints_matches
(the reference's sfm/import_feature_matches.py:76-104) on a COLMAP database created by the reference's own
COLMAPDatabase (sfm/colmap_utils/database.py), with `traj_to_matches` replaced by a function that returns the
match data of tests/golden/handoff_small.npz's trajectories (the reference function reads trajectory FILES; the
rest — keypoint shift, pair de-duplication, blobs — runs unmodified).  Needs a ParticleSfM checkout at $PSFM_REFERENCE:
    python tests/golden/make_import_golden.py
"""
import os
import sqlite3
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(os.environ["PSFM_REFERENCE"], "sfm"))
sys.path.insert(0, os.environ["PSFM_REFERENCE"])


def main():
    from particlesfm_b200 import handoff
    g = np.load(os.path.join(HERE, "handoff_small.npz"))
    off = np.concatenate([[0], np.cumsum(g["track_len"])])
    trajs = {int(k): {"locations": g["track_locs"][off[i]:off[i + 1]].tolist(),
                      "labels": g["track_labels"][off[i]:off[i + 1]].tolist(),
                      "frame_ids": g["track_frames"][off[i]:off[i + 1]].tolist()}
             for i, k in enumerate(g["track_keys"])}
    num_images = int(g["num_images"])
    names = ["%05d.png" % i for i in range(num_images)]
    data = handoff.traj_to_matches(trajs, num_images).as_reference(names)      # bit-exact vs the reference (test_handoff.py)
    # the reference module imports cv2-free helpers only; stub what it does not need here
    for mod in ("pycolmap",):
        sys.modules.setdefault(mod, types.ModuleType(mod))
    import import_feature_matches as ref
    from colmap_utils.database import COLMAPDatabase
    ref.traj_to_matches = lambda *a, **k: data
    out = {}
    for skip in (False, True):
        with tempfile.TemporaryDirectory() as td:
            path = os.path.join(td, "database.db")
            db = COLMAPDatabase.connect(path)
            db.create_tables()
            cam = db.add_camera(0, 64, 48, np.array([50.0, 32.0, 24.0]))
            # database ids deliberately NOT in name order: exercises the column flip of add_matches
            order = list(reversed(range(num_images)))
            for i in order:
                db.add_image(names[i], cam)
            db.commit()
            db.close()
            image_ids = ref.get_image_ids(path)
            ref.import_keypoints_matches(image_ids, "unused", path, "unused", "unused", skip_geometric_verification=skip)
            con = sqlite3.connect(path)
            tag = "skip" if skip else "verify"
            out[tag + "_keypoints"] = np.array([(i, r, c, bytes(b)) for i, r, c, b in con.execute("SELECT image_id, rows, cols, data FROM keypoints ORDER BY rowid")], dtype=object)
            out[tag + "_matches"] = np.array([(i, r, c, bytes(b)) for i, r, c, b in con.execute("SELECT pair_id, rows, cols, data FROM matches ORDER BY rowid")], dtype=object)
            out[tag + "_two_view"] = np.array([(i, r, c, bytes(b), cfg, bytes(F), bytes(E), bytes(H)) for i, r, c, b, cfg, F, E, H in
                                               con.execute("SELECT pair_id, rows, cols, data, config, F, E, H FROM two_view_geometries ORDER BY rowid")], dtype=object)
            out["image_names"] = np.array(list(image_ids.keys()), dtype=object)
            out["image_id_values"] = np.array(list(image_ids.values()), dtype=np.int64)
            con.close()
    np.savez_compressed(os.path.join(HERE, "import_small.npz"), **out)
    print({k: (v.shape if hasattr(v, "shape") else v) for k, v in out.items()})


if __name__ == "__main__":
    main()
