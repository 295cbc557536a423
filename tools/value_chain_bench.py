"""UDF value chain timing: exact-fp32 FFMA layers (chain mask without bit 1) against three bf16 planes on the tensor cores
(bit 1 set), at the C2 step's point count.  One JSON line.

    python tools/value_chain_bench.py [--points 65536] [--rounds 5] [--iters 20]

Per layer of the 8 x 256 UDF network (dense_forward against dense_forward_tc with a 3-plane image; the last layer as its
256 feature rows) and for the whole chain through UDFNetwork: the full forward with its saved context (`forward`) and the
value-only sweep (`udf_values`).  The two configurations alternate within every round in one process; each figure is the
median over the rounds of the CUDA-event time of `iters` back-to-back calls, with the min and max beside it.  Reported
with the device name and power limit read in the same run.  Requires a CUDA device; writes nothing.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

MASKS = {"ffma": 254, "tc3": 255}


def event_ms(fn, iters):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def stats(runs):
    import numpy as np
    return {"median_us": round(float(np.median(runs)) * 1e3, 1), "min_us": round(min(runs) * 1e3, 1),
            "max_us": round(max(runs) * 1e3, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=65536)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("value_chain_bench: needs a CUDA device")
    from neuraludf_b200 import _lib as L
    from neuraludf_b200 import synthetic as S
    from neuraludf_b200.models import fields as F
    from tools.eval_bench import power_limit
    lib = L.lib()
    dev = torch.device("cuda", 0)
    P = args.points
    cfg = S.udf_cfg()
    params = S.make_udf_params(cfg, 0)
    udf = F.UDFNetwork(d_in=3, d_out=cfg["d_out"], d_hidden=cfg["d_hidden"], n_layers=cfg["n_layers"], skip_in=cfg["skip_in"],
                       multires=cfg["multires"], bias=cfg["bias"], scale=cfg["scale"], geometric_init=True, weight_norm=True,
                       udf_type="abs")
    udf.load_state_dict(params)
    udf = udf.to(dev)
    x = (torch.rand(P, 3, generator=torch.Generator().manual_seed(0)) * 2 - 1).to(dev)
    st = L.stream_ptr()
    old_engine, old_mask = lib.nudf_get_engine(), lib.nudf_get_tc_mask()
    lib.nudf_set_engine(1)

    # one layer at a time: Y = softplus100(X W^T + b) (the last layer: its 256 feature rows, no activation)
    layers = []
    n_lin = len(cfg["layers"])
    for l, (k, n) in enumerate(cfg["layers"]):
        g, v = params["lin%d.weight_g" % l], params["lin%d.weight_v" % l]
        W = (g * v / v.norm(dim=1, keepdim=True)).float()
        b = params["lin%d.bias" % l].float()
        act = 2
        if l == n_lin - 1:
            W, b, n, act = W[1:], b[1:], n - 1, 0
        W, b = W.contiguous().to(dev), b.contiguous().to(dev)
        img = torch.zeros(lib.nudf_tc_image_elems(n, k, 3), dtype=torch.int16, device=dev)
        L.check(lib.nudf_tc_prepare_weights(L.ptr(W), k, n, k, 0, 3, L.ptr(img), st), "prepare_weights")
        X = torch.rand(P, k, device=dev)
        Y = torch.empty(P, n, device=dev)
        layers.append(dict(name="lin%d" % l, N=n, K=k, calls={
            "ffma": lambda X=X, W=W, b=b, Y=Y, n=n, k=k, act=act:
                lib.nudf_dense_forward(L.ptr(X), k, L.ptr(W), k, L.ptr(b), L.ptr(Y), n, P, n, k, act, st),
            "tc3": lambda X=X, img=img, b=b, Y=Y, n=n, k=k, act=act:
                lib.nudf_dense_forward_tc(L.ptr(X), k, L.ptr(img), 3, L.ptr(b), L.ptr(Y), n, P, n, k, act, st)}))

    chain = {"forward": lambda: udf(x), "udf_values": lambda: udf.udf_values(x)}
    runs = {}
    try:
        with torch.no_grad():
            for _ in range(args.rounds):
                for cfg_name, mask in MASKS.items():
                    lib.nudf_set_tc_mask(mask)
                    for lay in layers:
                        call = lay["calls"][cfg_name]
                        call()
                        runs.setdefault((lay["name"], cfg_name), []).append(event_ms(call, args.iters))
                    for name, fn in chain.items():
                        fn()                                       # refolds the weights for this mask
                        torch.cuda.synchronize()
                        runs.setdefault((name, cfg_name), []).append(event_ms(fn, args.iters))
    finally:
        lib.nudf_set_engine(old_engine)
        lib.nudf_set_tc_mask(old_mask)

    out = {"device": torch.cuda.get_device_name(0), "power_limit": power_limit(), "points": P, "rounds": args.rounds,
           "iters": args.iters, "masks": MASKS, "layers": {}, "chain": {}}
    for lay in layers:
        rec = {"N": lay["N"], "K": lay["K"]}
        for c in MASKS:
            rec[c] = stats(runs[(lay["name"], c)])
        rec["tc3_algorithmic_tflops"] = round(2.0 * P * lay["N"] * lay["K"] / (rec["tc3"]["median_us"] * 1e-6) / 1e12, 1)
        rec["speedup"] = round(rec["ffma"]["median_us"] / rec["tc3"]["median_us"], 2)
        out["layers"][lay["name"]] = rec
    for name in chain:
        rec = {c: stats(runs[(name, c)]) for c in MASKS}
        rec["speedup"] = round(rec["ffma"]["median_us"] / rec["tc3"]["median_us"], 2)
        rec["tc3_Mpts_per_s"] = round(P / (rec["tc3"]["median_us"] * 1e-6) / 1e6, 1)
        rec["ffma_Mpts_per_s"] = round(P / (rec["ffma"]["median_us"] * 1e-6) / 1e6, 1)
        out["chain"][name] = rec
    print(json.dumps(out))


if __name__ == "__main__":
    main()
