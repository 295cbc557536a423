"""DTU mesh-cleaning timing at full scan size: one JSON line.

    python tools/clean_bench.py [--faces 770000] [--repeats 5] [--no-reference]

Inputs: 49 views of 1600 x 1200 binary masks (silhouettes of a 96 mm sphere under a ring of cameras, written as PNGs to a
temporary scan directory) and a UV sphere of radius 100 mm with ~770 k faces (a 512^3 reconstruction's face count) plus
floating sheets, jittered by 0.8 mm.  Reported: the device name and power limit read in the same run; the host time of
load_dtu_scan (PNG decode of the 49 masks) and of their upload; device milliseconds (CUDA events, median of the repeats
after one warm-up) of the mask-pass dilation (k = 11), the visual-hull dilation (k = 31), one view vote over all vertices,
the face filter and compaction, and the whole clean_dtu_mesh from uploaded masks; vertex and face counts per stage; and --
unless --no-reference, when the reference's script is staged (oracle/ref_clean.py) -- the host wall time of the reference's
clean_mesh_faces_by_mask and clean_mesh_faces_by_visualhull on the same inputs, with whether their output equals ours.
Writes nothing outside a temporary directory.
"""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--faces", type=int, default=770_000)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--no-reference", action="store_true")
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("clean_bench needs a CUDA device")
    from neuraludf_b200 import clean as CL
    from oracle import ref_clean
    from tests.proto import clean_cases as C
    from tests.proto import eval_cases as EC
    from tools.eval_bench import power_limit
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(0)
    mats = C.ring(49, seed=0)
    masks = np.stack([C.silhouette(P, (0., 0., 0.), 96.0) for P in mats])
    n = int(round((args.faces / 2) ** 0.5))
    v, f = EC.uv_sphere(100.0, n, n)
    jv, jf = C.junk_sheets(rng)
    verts = np.concatenate([v, jv]) + rng.normal(scale=0.8, size=(len(v) + len(jv), 3))
    faces = np.concatenate([f, jf + len(v)])
    out = {"device": torch.cuda.get_device_name(0), "power_limit": power_limit(), "views": 49, "height": C.H, "width": C.W,
           "vertices": int(len(verts)), "faces": int(len(faces))}
    with tempfile.TemporaryDirectory() as tmp:
        ref_clean.write_scan(tmp, C.SCAN, mats, masks)
        t = time.perf_counter()
        _, loaded = CL.load_dtu_scan(tmp, C.SCAN)
        out["host_decode_ms"] = round(1e3 * (time.perf_counter() - t), 1)
    assert np.array_equal(loaded, masks)
    torch.cuda.synchronize()
    t = time.perf_counter()
    md = torch.from_numpy(loaded).to(dev)
    torch.cuda.synchronize()
    out["upload_ms"] = round(1e3 * (time.perf_counter() - t), 1)
    vd, fd = torch.from_numpy(verts).to(dev), torch.from_numpy(faces).to(dev)
    runs = []
    for rep in range(args.repeats + 1):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)]
        ev[0].record()
        packed = CL.dilate_masks(md, 11)
        ev[1].record()
        CL.dilate_masks(md, 31, below=True)
        ev[2].record()
        counts = CL.count_views(vd, mats, packed, C.H, C.W)
        ev[3].record()
        CL.clean_mesh(vd, fd, counts > 2)
        ev[4].record()
        stages = CL.clean_dtu_mesh(vd, fd, mats, md)
        ev[5].record()
        torch.cuda.synchronize()
        if rep:
            runs.append([ev[i].elapsed_time(ev[i + 1]) for i in range(5)])
    ms = np.median(np.array(runs), axis=0)
    out["ms"] = dict(zip(["dilate_k11", "dilate_k31", "vote", "compact", "clean_dtu_mesh"], [round(float(x), 3) for x in ms]))
    out["stage_sizes"] = [[int(s[0].shape[0]), int(s[1].shape[0])] for s in stages]
    if not args.no_reference and (ref_clean.verify() or ref_clean.stage(verbose=False) is not None):
        ref = ref_clean.run_clean(verts, faces, mats, masks, scan=C.SCAN, imgs_idx=None)
        out["reference_s"] = [round(s["seconds"], 2) for s in ref]
        out["reference_cpu_count"] = os.cpu_count()
        out["reference_equal"] = all(np.array_equal(s["verts"], g[0].cpu().numpy()) and np.array_equal(s["faces"], g[1].cpu().numpy())
                                     for s, g in zip(ref, stages))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
