"""Timing of the tensor-core weight-gradient contraction (nudf_wgrad, engine 1: gemm_tn_kernel and its fixed-order split-K
reduction) at each shape the C2 step runs it at, dW[n_out, n_in] += dZ[P, n_out]^T X[P, n_in].  One JSON line.

    python tools/wgrad_bench.py [--points 65536] [--rounds 5] [--iters 20]

Each figure is the median over the rounds of the CUDA-event time of `iters` back-to-back calls, with the min and max
beside it.  The algorithmic rate counts 2 P n_out n_in flops (the kernel issues three bf16 products per multiply-add);
the bandwidth counts the two fp32 operands read once, 4 P (n_out + n_in) bytes.  The kernel stages each operand block once
per CTA that needs it: every 128-row block of dZ for each 128-column tile of n_in, and the other way round, so
`l2_to_sm_GB_per_s` counts 4 P (ceil(n_in / 128) n_out + ceil(n_out / 128) n_in) bytes (widths rounded up to 4 floats,
the whole float4s a ragged tile copies) going from L2 to the SMs.  The operands have the row strides the networks give
them (widths rounded up to 8 floats, 16-byte-aligned rows).  `per_step_us` weighs each shape by the
number of contractions of that shape in one C2 step (25).  The calls carry no bias column sums, which the step's
contractions fuse into the same kernel.  Compare two builds of the library by running this in separate processes with
NUDF_LIB_PATH pointing at each; the library path is part of the output, with the device name and power limit read in
the same run.  Requires a CUDA device; writes nothing.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

# (n_out, n_in): contractions per C2 step.  UDF (17): tangent chain D_l^T Adot_l for layers 0-7, backward chain
# Zbar_l^T A_l for layers 0-7 and the 256 feature rows of layer 8.  Colour (8): the base and main stacks' first layers
# (259 and 158 inputs) and three 128 x 128 hidden layers each.
C2_SHAPES = {(256, 256): 13, (256, 39): 2, (217, 256): 2, (128, 128): 6, (128, 158): 1, (128, 259): 1}
TILE = 128


def ld8(n):
    return (n + 7) // 8 * 8


def l2_to_sm_bytes(P, n_out, n_in):
    """bytes staged into shared memory: each CTA of the (n_out / 128) x (n_in / 128) tile grid reads its two blocks"""
    r4 = lambda n: (n + 3) // 4 * 4
    tiles = lambda n: (n + TILE - 1) // TILE
    return 4 * P * (tiles(n_in) * r4(n_out) + tiles(n_out) * r4(n_in))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=65536)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("wgrad_bench: needs a CUDA device")
    from neuraludf_b200 import _lib as L
    from tools.eval_bench import power_limit
    from tools.value_chain_bench import event_ms, stats
    lib = L.lib()
    dev = torch.device("cuda", 0)
    P = args.points
    g = torch.Generator(device=dev).manual_seed(0)
    st = L.stream_ptr()
    calls = {}
    for (n_out, n_in) in C2_SHAPES:
        dZ = torch.randn(P, ld8(n_out), generator=g, device=dev)
        X = torch.randn(P, ld8(n_in), generator=g, device=dev)
        dW = torch.zeros(n_out, n_in, device=dev)
        calls[(n_out, n_in)] = (dZ, X, dW, lambda dZ=dZ, X=X, dW=dW, n_out=n_out, n_in=n_in: L.check(
            lib.nudf_wgrad(L.ptr(dZ), dZ.stride(0), L.ptr(X), X.stride(0), n_out, n_in, P, L.ptr(dW), n_in, 1, st),
            "wgrad"))
    for *_, fn in calls.values():
        fn()
    torch.cuda.synchronize()
    runs = {k: [] for k in calls}
    for _ in range(args.rounds):
        for k, (*_, fn) in calls.items():
            runs[k].append(event_ms(fn, args.iters))

    out = {"lib": os.path.abspath(L.LIB_PATH), "device": torch.cuda.get_device_name(0), "power_limit": power_limit(),
           "points": P, "rounds": args.rounds, "iters": args.iters, "shapes": {}}
    per_step = 0.0
    for (n_out, n_in), count in C2_SHAPES.items():
        rec = stats(runs[(n_out, n_in)])
        t = rec["median_us"] * 1e-6
        nbytes = 4 * P * (n_out + n_in)
        rec["count_per_step"] = count
        rec["algorithmic_tflops"] = round(2.0 * P * n_out * n_in / t / 1e12, 1)
        rec["operand_GB_per_s"] = round(nbytes / t / 1e9, 1)
        rec["l2_to_sm_GB_per_s"] = round(l2_to_sm_bytes(P, n_out, n_in) / t / 1e9, 1)
        out["shapes"]["%dx%d" % (n_out, n_in)] = rec
        per_step += count * rec["median_us"]
    out["per_step_us"] = round(per_step, 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
