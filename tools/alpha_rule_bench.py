"""CUDA-event timings of the two sdf2alpha rules: compositing forward, compositing backward and one up-sampling round, at
the C2 shape (512 rays x 128 samples) and at the DTU conf's fine-pass shape (512 rays x 114 samples + 32 NeRF++
columns; up-sampling on the 64 coarse samples).  Both rules run in one process, alternated, on the same seeded inputs.

    python tools/alpha_rule_bench.py [--iters 200] [--repeats 5]

Prints the card's name and power limit, then one JSON line per (shape, stage, rule) with the median and spread over the
repeats.  Writes nothing."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from neuraludf_b200 import ops  # noqa: E402
from tests.test_raymath_host import make_case  # noqa: E402

SHAPES = {"C2": (512, 128, 0, 64), "DTU": (512, 114, 32, 64)}   # rays, samples, outside columns, coarse samples


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                            capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        pl = "unknown"
    return name, pl


def inputs(N, S, Oo, seed=1):
    reps = -(-N // 6)
    cs = [make_case(seed + k, S, Oo, True) for k in range(reps)]
    cat = lambda k: torch.cat([c[k] for c in cs])[:N].float().cuda().contiguous()
    P = N * S
    a = dict(udf=cat("udf").reshape(P), grads=cat("grads").reshape(P, 3), scb=cat("scb").reshape(P, 3),
             sc=cat("sc").reshape(P, 3), bga=cat("bga") if Oo else None, bgc=cat("bgc") if Oo else None,
             heads=torch.tensor([403.4, 148.4, 20.1], device="cuda"))
    geom = (cat("d"), cat("pts").reshape(P, 3), cat("mid"), cat("dists"))
    return a, geom, cat("o"), cat("z"), float(cs[0]["dists"][0, -1])


def timed(fn, iters):
    fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / iters   # us per call


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("alpha_rule_bench needs a CUDA device")
    name, pl = card()
    print(json.dumps({"card": name, "power_limit_and_max_sm_clock": pl}), flush=True)
    for shape, (N, S, Oo, n0) in SHAPES.items():
        args, geom, o, z, sd = inputs(N, S, Oo)
        d = geom[0]
        zc = z[:, ::max(1, S // n0)][:, :n0].contiguous()
        uc = args["udf"].reshape(N, S)[:, ::max(1, S // n0)][:, :n0].contiguous()
        stages = {}
        for rule in (0, 1):
            cfg = ops._make_cfg(N, S, Oo, sd, 0.5, 0.3, 25000.0, False, None, rule)
            leaves = {k: (v.clone().requires_grad_(True) if v is not None else None) for k, v in args.items()}

            def fwd(cfg=cfg, leaves=leaves):
                with torch.no_grad():
                    ops.composite(leaves["udf"], leaves["grads"], leaves["scb"], leaves["sc"], leaves["bga"],
                                  leaves["bgc"], leaves["heads"], geom, cfg, want_diag=False)

            comp = ops.composite(leaves["udf"], leaves["grads"], leaves["scb"], leaves["sc"], leaves["bga"],
                                 leaves["bgc"], leaves["heads"], geom, cfg, want_diag=False)
            loss = comp["color"].sum() + comp["depth"].sum() + comp["ray_sums"].sum()

            def bwd(loss=loss, leaves=leaves):
                torch.autograd.grad(loss, [leaves["udf"], leaves["heads"]], retain_graph=True)

            def up(rule=rule):
                ops.up_sample(0, o, d, zc, uc, sd, 16, 64 * 2 ** 4, 64 * 2 ** 5, 20.0, alpha_rule=rule)

            stages[rule] = {"composite_forward": fwd, "composite_backward_autograd": bwd, "up_sample_round": up}
        res = {(st, r): [] for r in (0, 1) for st in stages[0]}
        for _ in range(a.repeats):
            for st in stages[0]:
                for r in (0, 1):                       # alternate the rules inside every repeat
                    res[(st, r)].append(timed(stages[r][st], a.iters))
        for (st, r), v in res.items():
            v = sorted(v)
            print(json.dumps({"shape": shape, "rays": N, "samples": S, "outside": Oo, "stage": st,
                              "rule": ["numerical", "theorical"][r], "median_us": round(v[len(v) // 2], 2),
                              "min_us": round(v[0], 2), "max_us": round(v[-1], 2)}), flush=True)
    torch.cuda.synchronize()


if __name__ == "__main__":
    main()
