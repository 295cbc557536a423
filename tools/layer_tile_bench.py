"""Per-layer timing of the tensor-core layer kernel: one 2-plane and one 3-plane 256 x 256 layer (Y = X W^T + b) through
nudf_dense_forward_tc at the C2 step's point count.  One JSON line.

    python tools/layer_tile_bench.py [--points 65536] [--rounds 5] [--iters 50]

Each figure is the median over the rounds of the CUDA-event time of `iters` back-to-back calls, with the min and max
beside it.  The achieved bandwidth counts the bytes the layer needs, from the shapes: the fp32 activations read once,
the fp32 output written once, the bias and the weight image read once.  Compare two builds of the library by running
this in separate processes with NUDF_LIB_PATH pointing at each; the library path is part of the output, with the device
name and power limit read in the same run.  Requires a CUDA device; writes nothing.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=65536)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("layer_tile_bench: needs a CUDA device")
    from neuraludf_b200 import _lib as L
    from tools.eval_bench import power_limit
    from tools.value_chain_bench import event_ms, stats
    lib = L.lib()
    dev = torch.device("cuda", 0)
    P, N, K = args.points, 256, 256
    g = torch.Generator().manual_seed(0)
    X = torch.randn(P, K, generator=g).to(dev)
    W = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev)
    b = torch.randn(N, generator=g).to(dev)
    Y = torch.empty(P, N, device=dev)
    st = L.stream_ptr()
    calls = {}
    for planes in (2, 3):
        img = torch.zeros(lib.nudf_tc_image_elems(N, K, planes), dtype=torch.int16, device=dev)
        L.check(lib.nudf_tc_prepare_weights(L.ptr(W), K, N, K, 0, planes, L.ptr(img), st), "prepare_weights")
        calls[planes] = (img, lambda img=img, planes=planes: L.check(
            lib.nudf_dense_forward_tc(L.ptr(X), K, L.ptr(img), planes, L.ptr(b), L.ptr(Y), N, P, N, K, 0, st), "dense_forward_tc"))
    runs = {planes: [] for planes in calls}
    for planes, (_, fn) in calls.items():
        fn()
    torch.cuda.synchronize()
    for _ in range(args.rounds):
        for planes, (_, fn) in calls.items():
            runs[planes].append(event_ms(fn, args.iters))

    out = {"lib": os.path.abspath(L.LIB_PATH), "device": torch.cuda.get_device_name(0), "power_limit": power_limit(),
           "points": P, "N": N, "K": K, "rounds": args.rounds, "iters": args.iters, "layers": {}}
    for planes, (img, _) in calls.items():
        rec = stats(runs[planes])
        nbytes = 4 * P * K + 4 * P * N + 4 * N + 2 * img.numel()
        rec["bytes"] = nbytes
        rec["achieved_GB_per_s"] = round(nbytes / (rec["median_us"] * 1e-6) / 1e9, 1)
        rec["algorithmic_tflops"] = round(2.0 * P * N * K / (rec["median_us"] * 1e-6) / 1e12, 1)
        out["layers"]["planes%d" % planes] = rec
    print(json.dumps(out))


if __name__ == "__main__":
    main()
