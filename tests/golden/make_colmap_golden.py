"""Writes tests/golden/colmap_model/{cameras,images,points3D}.bin with the REFERENCE's own
writer (the reference's sfm/colmap_utils/read_write_model.py:447-456, imported read-only) from
the values of colmap_model_def.py, and checks that the reference's reader gets them back.

    PSFM_REFERENCE=/path/to/particle-sfm python tests/golden/make_colmap_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(os.environ["PSFM_REFERENCE"], "sfm", "colmap_utils"))


def main():
    import read_write_model as ref
    from colmap_model_def import model_values
    cams, imgs, pts = model_values()
    rc = {i: ref.Camera(id=i, model=ref.CAMERA_MODEL_IDS[c["model_id"]].model_name, width=c["width"], height=c["height"],
                        params=c["params"]) for i, c in cams.items()}
    ri = {i: ref.Image(id=i, qvec=m["qvec"], tvec=m["tvec"], camera_id=m["camera_id"], name=m["name"], xys=m["xys"],
                       point3D_ids=m["point3D_ids"]) for i, m in imgs.items()}
    rp = {i: ref.Point3D(id=i, xyz=p["xyz"], rgb=p["rgb"], error=p["error"], image_ids=p["image_ids"],
                         point2D_idxs=p["point2D_idxs"]) for i, p in pts.items()}
    out = os.path.join(HERE, "colmap_model")
    os.makedirs(out, exist_ok=True)
    ref.write_model(rc, ri, rp, out, ext=".bin")
    c2, i2, p2 = ref.read_model(out, ext=".bin")
    assert list(c2) == list(rc) and list(i2) == list(ri) and list(p2) == list(rp)
    assert all(np.array_equal(i2[k].xys, ri[k].xys) for k in ri)
    print({f: os.path.getsize(os.path.join(out, f)) for f in sorted(os.listdir(out))})


if __name__ == "__main__":
    main()
