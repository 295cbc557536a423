"""Per-layer timing of the tensor-core layer kernel (Y = X W^T + b) through nudf_dense_forward_tc at the C2 step's
point count: the 2-plane layer at 256 x 256 and 128 x 128, and the 3-plane layer at 256 x 256, 128 x 128 and 256 x 39
(the UDF network's first layer).  One JSON line.

    python tools/layer_tile_bench.py [--points 65536] [--rounds 5] [--iters 50]

Each activation has a row stride of K rounded up to 4 floats and a 16-byte-aligned base, as the networks' operands
have: the kernels read it through a tensor map, with no repack.  Each figure is the median over the rounds of the CUDA-event time of `iters` back-to-back calls, with the min and max beside
it; the layers alternate within each round.  The achieved bandwidth counts the bytes the layer needs, from
the shapes: the fp32 activations read once, the fp32 output written once, the bias and the weight image read once.
Compare two builds of the library by running this in separate processes with NUDF_LIB_PATH pointing at each; the
library path is part of the output, with the device name, power limit and SM clock read in the same run.  Requires a
CUDA device; writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def sm_clock():
    """current / maximum SM clock of device 0 (MHz), read right after the timed work"""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


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
    P = args.points
    g = torch.Generator().manual_seed(0)
    st = L.stream_ptr()
    calls = {}    # name -> (bytes, flops, fn)

    def add(name, N, K, planes):
        ld = (K + 3) // 4 * 4
        X = torch.zeros(P, ld, device=dev)
        X[:, :K] = torch.randn(P, K, generator=g).to(dev)
        W = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev)
        b = torch.randn(N, generator=g).to(dev)
        Y = torch.empty(P, N, device=dev)
        img = torch.zeros(lib.nudf_tc_image_elems(N, K, planes), dtype=torch.int16, device=dev)
        L.check(lib.nudf_tc_prepare_weights(L.ptr(W), K, N, K, 0, planes, L.ptr(img), st), "prepare_weights")
        fn = lambda: L.check(lib.nudf_dense_forward_tc(L.ptr(X), ld, L.ptr(img), planes, L.ptr(b), L.ptr(Y), N, P, N, K, 0, st),
                             "dense_forward_tc")
        calls[name] = (4 * P * K + 4 * P * N + 4 * N + 2 * img.numel(), 2.0 * P * N * K, fn, (X, W, b, Y, img))

    for n in (256, 128):
        add("planes2_%dx%d_ring" % (n, n), n, n, 2)
    add("planes3_256x256_tma", 256, 256, 3)
    add("planes3_128x128_tma", 128, 128, 3)
    add("planes3_256x39_tma", 256, 39, 3)
    runs = {name: [] for name in calls}
    for _, _, fn, _ in calls.values():
        fn()
    torch.cuda.synchronize()
    for _ in range(args.rounds):
        for name, (_, _, fn, _) in calls.items():
            runs[name].append(event_ms(fn, args.iters))
    clock = sm_clock()

    out = {"lib": os.path.abspath(L.LIB_PATH), "device": torch.cuda.get_device_name(0), "power_limit": power_limit(),
           "sm_clock_MHz_cur_max": clock, "points": P, "rounds": args.rounds, "iters": args.iters, "layers": {}}
    for name, (nbytes, flops, _, _) in calls.items():
        rec = stats(runs[name])
        rec["bytes"] = nbytes
        rec["achieved_GB_per_s"] = round(nbytes / (rec["median_us"] * 1e-6) / 1e9, 1)
        rec["algorithmic_tflops"] = round(flops / (rec["median_us"] * 1e-6) / 1e12, 1)
        out["layers"][name] = rec
    print(json.dumps(out))


if __name__ == "__main__":
    main()
