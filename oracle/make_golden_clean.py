"""Golden mesh cleanings of the reference script -- tests/golden/clean_<case>.NN.npz.

    python oracle/make_golden_clean.py      # needs the reference checkout (oracle/ref_clean.py stages its script)

Cases (tests/proto/clean_cases.py): a sphere with floating sheets under a ring of cameras and binary masks; anti-aliased
masks (every value around 128) at kernel 1; projections onto the image border, the visual-hull border, behind the camera
and at the camera centre at the even kernel 10; kernel 31; all 49 views (imgs_idx=None).  The reference runs unmodified
under oracle/ref_clean.py's trimesh stub, its second stage fed the first stage's export.  Stored per case and stage: the
view counts, the SHA-256 of the thresholded dilated masks packed as csrc/mesh_clean.cu packs them, and the SHA-256 and sizes
of the exported vertices (float64) and faces (int64); for the inputs, the SHA-256 of the regenerated vertices, faces,
matrices and masks.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_clean  # noqa: E402
from tests.golden_util import save_fixtures  # noqa: E402
from tests.proto import clean_cases as C  # noqa: E402
from tests.proto import mesh_clean as M  # noqa: E402


def main():
    if not ref_clean.verify() and ref_clean.stage() is None:
        sys.exit("the reference checkout is required (oracle/ref_clean.py)")
    for name in C.CASES:
        c = C.case(name)
        stages = ref_clean.run_clean(c["verts"], c["faces"], c["mats"], c["masks"], scan=C.SCAN, imgs_idx=c["imgs_idx"],
                                     mask_kernel=c["mask_kernel"], minimal_vis=c["minimal_vis"])
        out = dict(inputs_sha=np.array(C.sha256(c["verts"], c["faces"], c["mats"], c["masks"])),
                   params=np.array([c["mask_kernel"], c["minimal_vis"], -1 if c["imgs_idx"] is None else len(c["imgs_idx"])]))
        for tag, below, s in (("mask", False, stages[0]), ("hull", True, stages[1])):
            out["counts_" + tag] = s["counts"].astype(np.int32)
            out["packed_sha_" + tag] = np.array(C.sha256(M.pack(M.threshold(s["dilated"], below))))
            out["out_sha_" + tag] = np.array(C.sha256(np.asarray(s["verts"], np.float64), np.asarray(s["faces"], np.int64)))
            out["out_size_" + tag] = np.array([len(s["verts"]), len(s["faces"])])
        save_fixtures("clean_" + name, out)
        print(name, "vertices", len(c["verts"]), "->", out["out_size_mask"].tolist(), "->", out["out_size_hull"].tolist())


if __name__ == "__main__":
    main()
