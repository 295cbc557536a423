"""Golden point-cloud evaluations of the reference scripts -- tests/golden/eval_<case>.NN.npz.

    python oracle/make_golden_eval.py       # needs the reference checkout (oracle/ref_eval.py stages its scripts)

Cases (tests/proto/eval_cases.py): a closed mesh in mm with GT partly off-surface and partly below the plane and an ObsMask
with holes; an open patch whose GT extends past it (s2d >= max_dist); `--mode pcd`; DeepFashion scale (density 0.002).  The
DTU cases run `eval_cloud(args)`, DeepFashion its `__main__` block, both unmodified under oracle/ref_eval.py's open3d stub
with a seeded, recorded shuffle.  Stored per case: the inputs, the sampled cloud before the shuffle, the permutation, the
kept positions, the DTU in-bound / in-obs / above sets, both distance arrays, the means, the vis colours and (DeepFashion)
the printed metrics and the log.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_eval  # noqa: E402
from tests.golden_util import save_fixtures  # noqa: E402
from tests.proto import eval_cases as C  # noqa: E402


def _mask_of(sub, full):
    """boolean mask m over the rows of `full` with full[m] == sub, rows taken in order (sub is an ordered subset)"""
    m = np.zeros(len(full), bool)
    j = 0
    for i in range(len(full)):
        if j < len(sub) and np.array_equal(full[i], sub[j]):
            m[i] = True
            j += 1
    assert j == len(sub)
    return m


def main():
    if not ref_eval.verify() and ref_eval.stage() is None:
        sys.exit("the reference checkout is required (oracle/ref_eval.py)")
    for name in C.CASES:
        c = C.case(name)
        p = c["params"]
        faces = c["faces"]
        if c["protocol"] == "dtu":
            rec = ref_eval.run_dtu(c["data"], faces, c["gt"], c["obs_mask"], c["bb"], c["res"], c["plane"], c["seed"],
                                   density=p["density"], patch=p["patch"], max_dist=p["max_dist"], vis=p["vis"])
            (q1, d1), (q2, d2) = rec["kneighbors"]
            data_down, data_color = rec["vis"]["vis_001_d2gt.ply"]
            _, gt_color = rec["vis"]["vis_001_gt2d.ply"]
            data_in = rec["fits"][2]
            inbound = _mask_of(data_in, data_down)
            in_obs_index = np.nonzero(_mask_of(q1, data_down))[0]
            above = _mask_of(q2, c["gt"])
            out = dict(mean_d2s=rec["mean_d2s"], mean_s2d=rec["mean_s2d"], over_all=rec["over_all"], inbound=inbound,
                       in_obs_index=in_obs_index, above=above)
            inputs = dict(obs_mask=c["obs_mask"], bb=c["bb"], res=c["res"], plane=c["plane"])
        else:
            rec = ref_eval.run_deepfashion(c["data"], faces, c["gt"], c["seed"], density=p["density"], max_dist=p["max_dist"],
                                           vis=p["vis"])
            (q1, d1), (q2, d2) = rec["kneighbors"]
            data_down, data_color = rec["vis"]["vis_300_d2gt.ply"]
            _, gt_color = rec["vis"]["vis_300_gt2d.ply"]
            pr = rec["printed"]
            out = dict(mean_d2s=pr["mean_d2gt"], mean_s2d=pr["mean_gt2d"], over_all=pr["over_all"],
                       printed=np.array([pr[k] for k in ("precision_1mm", "recall_1mm", "fscore_1mm", "precision_2mm",
                                                         "recall_2mm", "fscore_2mm")]), log=np.array(rec["log"]))
            inputs = {}
        assert np.array_equal(rec["data_pcd"][rec["perm"]][rec["kept_index"]], data_down)
        save_fixtures("eval_" + name, dict(
            inputs, data=c["data"], gt=c["gt"], seed=c["seed"], params=np.array([p["density"], p.get("patch", 0.0),
                                                                                   p["max_dist"], p["vis"]]),
            **({"faces": faces} if faces is not None else {}),
            data_pcd=rec["data_pcd"], perm=rec["perm"], kept_index=rec["kept_index"], dist_d2s=d1[:, 0], dist_s2d=d2[:, 0],
            data_color=data_color, gt_color=gt_color, **out))
        print(name, "points", len(rec["data_pcd"]), "kept", len(rec["kept_index"]), "d2s", len(d1), "s2d", len(d2),
              "s2d >= max", int((d2 >= p["max_dist"]).sum()), "over_all", out["over_all"])


if __name__ == "__main__":
    main()
