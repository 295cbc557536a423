"""Connected-component filter timing (neuraludf_b200/clean.py clean_outliers): one JSON line.

    python tools/cc_bench.py [--sizes 512 1024] [--strip 2000000] [--repeats 5]

Reported with the device name and power limit read in the same run.  Inputs: the C5 scene's band meshes after the vertex
filter at dist_threshold_ratio 5, built as tools/mesh_post_bench.py builds them, and a strip of --strip faces in random
face order (deep union-find trees).  Per input, the CUDA-event milliseconds of each stage of keep_largest (edge keys:
nudf_mp_faces; sort: torch.sort of the keys; labelling: nudf_cc_label; sizes and selection: bincount and argmax;
compaction: the submesh), of remove_small_components' sizes and selection, and of the whole clean_outliers in both branches
(the load merge included).  Median of the repeats after one warm-up.  `restatement_host_ms` is the NumPy / scipy
restatement (tests/proto/mesh_cc.py) of clean_outliers(keep_largest=True) on the host for the same input, checked to give
the same bits: it is not trimesh's time, which cannot be measured here.  Requires a CUDA device; writes nothing.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def stages(CL, v, f, repeats):
    """median CUDA-event ms of keep_largest's stages and of remove_small_components' selection"""
    import numpy as np
    import torch
    from neuraludf_b200.mesh_post import _face_pass
    names = ["edge_keys", "sort", "labelling", "sizes_selection", "compaction", "sizes_selection_faces_num"]
    runs = []
    for rep in range(repeats + 1):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(7)]
        ev[0].record()
        codes = _face_pass(v, f, None)[2]
        ev[1].record()
        keys, order = torch.sort(codes.reshape(-1) >> 1)
        key_face = order // 3
        ev[2].record()
        label, paired = CL._label_faces(keys, key_face, f.shape[0])
        ev[3].record()
        keep = CL._largest(label)
        ev[4].record()
        out = CL._submesh(v, f, keep)
        ev[5].record()
        CL._at_least(label, paired, CL.FACES_NUM)
        ev[6].record()
        torch.cuda.synchronize()
        if rep:
            runs.append([ev[i].elapsed_time(ev[i + 1]) for i in range(6)])
    med = np.median(np.array(runs), axis=0)
    return dict(zip(names, (round(float(x), 3) for x in med))), label, paired, out


def measure(CL, P, name, v64, faces, repeats):
    import numpy as np
    import torch
    from tools.mesh_band_bench import timed
    r3 = lambda x: round(float(x), 3)
    v, f = v64.contiguous(), faces.contiguous()
    ms, label, paired, (kv, kf) = stages(CL, v, f, repeats)
    rec = {"faces": int(f.shape[0]), "vertices": int(v.shape[0]), "ms": ms,
           "components": int((label == torch.arange(label.numel(), device=label.device)).sum()),
           "unpaired_faces": int((paired == 0).sum()), "largest_faces": int(kf.shape[0])}
    rec["ms"]["keep_largest_total"] = r3(sum(ms[k] for k in ("edge_keys", "sort", "labelling", "sizes_selection",
                                                              "compaction")))
    for tag, kl in (("clean_outliers_largest", True), ("clean_outliers_faces_num", False)):
        t, res = timed(lambda: CL.clean_outliers(v, f, keep_largest=kl), repeats)
        rec["ms"][tag] = r3(t)
        if kl:
            dv, df = res
    hv, hf = v.cpu().numpy(), f.cpu().numpy()
    t = time.perf_counter()
    pv, pf = P.clean_outliers(hv, hf, keep_largest=True)
    rec["restatement_host_ms"] = r3(1e3 * (time.perf_counter() - t))
    rec["restatement_same_bits"] = bool(np.array_equal(pf, df.cpu().numpy())
                                        and np.array_equal(pv.view(np.int64), dv.cpu().numpy().view(np.int64)))
    print(json.dumps({name: rec}), file=sys.stderr, flush=True)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="*", default=[512, 1024])
    ap.add_argument("--strip", type=int, default=2_000_000)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--ratio", type=float, default=5.0)
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("cc_bench needs a CUDA device")
    from neuraludf_b200 import clean as CL
    from neuraludf_b200 import grid, mesh
    from tests.golden_util import load_golden
    from tests.gpu_util import build_modules
    from tests.proto import mesh_cc as P
    from tools.eval_bench import power_limit
    out = {"device": torch.cuda.get_device_name(0), "power_limit": power_limit(), "scene": "C5 golden UDF network",
           "dist_threshold_ratio": args.ratio, "inputs": {}}
    dev = torch.device("cuda", 0)
    if args.sizes:
        udf = build_modules(load_golden(), "cuda")[0]
    for N in args.sizes:
        voxel = 2.0 / (N - 1)
        df, _ = grid.udf_band(udf, N)
        vi, faces = mesh._mc_lattice(udf, N, df, 0, 1 << 21)
        del df
        v64 = vi.double() * voxel - 1.0
        vd = udf.udf_values(v64.float()).reshape(-1)
        faces = faces[vd[faces].max(dim=1).values < voxel * args.ratio]
        del vi, vd
        torch.cuda.empty_cache()
        out["inputs"]["c5_%d" % N] = measure(CL, P, "c5_%d" % N, v64, faces, args.repeats)
        del v64, faces
        torch.cuda.empty_cache()
    if args.strip:
        v, f = P.strip(args.strip)
        f = f[np.random.default_rng(0).permutation(len(f))]
        out["inputs"]["strip_%d" % args.strip] = measure(CL, P, "strip", torch.from_numpy(v).to(dev),
                                                         torch.from_numpy(f).to(dev), args.repeats)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
