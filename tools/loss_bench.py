"""Times the device colour loss (neuraludf_b200.loss.ColorLoss) against the reference's unmodified loss/loss.py on the same
GPU, counts the kernels each launches per forward + backward, and times a fine-tuning step "render_core forward -> device
ColorLoss -> backward" eagerly and replayed as one CUDA graph.

    python tools/loss_bench.py [--rays 512] [--iters 50] [--out result.json]

Loss shapes: the fine-tuning conf's (confs/udf_dtu_blending_ft.conf: N = 512, h_patch_size = 5, SSIM; weights 0.01 / 1.0 /
0.1 / 0.1, pixel_mask present) and h = 3 NCC.  The step: the golden-scene-sized networks of neuraludf_b200.synthetic, 512
rays x 64 samples, render_core without blending (its blending path reads the host itself: the tool reports where), the
loss on render_core's color_base / color and an h = 3 NCC patch term on the rendered colour shifted by a fixed texture,
patch mask weight_sum > 0.5 as the runner forms it.  The reference loss cannot enter such a graph:
`int(penalize_ratio * mask.sum())` (loss.py:82) reads a device value on the host, which a stream capture forbids; the tool shows that read with
torch.cuda.set_sync_debug_mode("error") instead of attempting the capture.  The reference loss needs the staged reference
(oracle/make_ref.py).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

INPUTS = ["color_base", "color", "gt_color", "color_pixel", "pixel_mask", "patch_colors", "gt_patch_colors", "patch_mask"]
PREDS = ["color_base", "color", "color_pixel", "patch_colors"]
WEIGHTS = (0.01, 1.0, 0.1, 0.1)


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def timed(fn, iters, warmup=5):
    """median and min of per-call device time (CUDA events), ms"""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts), min(ts)


def count_launches(fn):
    """kernels and memcpy / memset operations of one call (torch.profiler, CUDA activities)"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    kernels = copies = 0
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        if "memcpy" in e.name.lower() or "memset" in e.name.lower():
            copies += 1
        else:
            kernels += 1
    return kernels, copies


def loss_inputs(n, h, dev, seed=0):
    rng = np.random.default_rng(seed)
    P = (2 * h + 1) ** 2
    f = lambda *s: torch.from_numpy(rng.random(s).astype(np.float32)).to(dev)  # noqa: E731
    gt = f(n, P, 3)
    t = {"gt_color": f(n, 3), "color_base": f(n, 3), "color": f(n, 3), "color_pixel": f(n, 3), "gt_patch_colors": gt,
         "patch_colors": (gt + 0.2 * (f(n, P, 3) - 0.5)).clamp(0, 1), "pixel_mask": (f(n, 1) > 0.3).float(),
         "patch_mask": f(n, 1) > 0.2}
    for k in PREDS:
        t[k].requires_grad_(True)
    return t


def loss_step(fn, t):
    def step():
        for k in PREDS:
            t[k].grad = None
        fn(*[t[k] for k in INPUTS])["loss"].backward()
    return step


def host_sync_error(step):
    """the error torch.cuda.set_sync_debug_mode('error') raises for `step`, or None when it runs without a host read"""
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        step()
        return None
    except RuntimeError as e:
        return str(e).splitlines()[0][:160]
    finally:
        torch.cuda.set_sync_debug_mode(0)
        torch.cuda.synchronize()


def bench_loss(args, dev, ref_mod):
    from neuraludf_b200.loss import ColorLoss
    rows = []
    for h, ptype in ((5, "ssim"), (3, "ncc")):
        t = loss_inputs(args.rays, h, dev)
        dev_fn = ColorLoss(*WEIGHTS, pixel_loss_type="l1", patch_loss_type=ptype, h_patch_size=h)
        row = {"rays": args.rays, "h": h, "type": ptype}
        step = loss_step(dev_fn, t)
        row["device_ms"], row["device_ms_min"] = timed(step, args.iters)
        row["device_kernels"], row["device_copies"] = count_launches(step)
        row["device_host_sync"] = host_sync_error(step)
        if ref_mod is not None:
            ref_fn = ref_mod.ColorLoss(*WEIGHTS, pixel_loss_type="l1", patch_loss_type=ptype, h_patch_size=h).to(dev)
            rstep = loss_step(ref_fn, t)
            row["reference_ms"], row["reference_ms_min"] = timed(rstep, args.iters)
            row["reference_kernels"], row["reference_copies"] = count_launches(rstep)
            row["reference_host_sync"] = host_sync_error(rstep)
        rows.append(row)
        print(json.dumps(row), flush=True)
    return rows


def bench_step(args, dev, ref_mod):
    """render_core forward -> ColorLoss -> backward, eager (device and reference loss) and as one replayed CUDA graph"""
    from neuraludf_b200 import synthetic as S
    from neuraludf_b200.loss import ColorLoss
    from neuraludf_b200.models import fields as F
    from neuraludf_b200.models.udf_renderer_blending import UDFRendererBlending
    udf_c, col_c = S.udf_cfg(), S.color_cfg()
    udf = F.UDFNetwork(d_in=3, d_out=257, d_hidden=256, n_layers=8, skip_in=(4,), multires=6, bias=0.5, scale=1.0,
                       geometric_init=True, weight_norm=True, udf_type="abs")
    udf.load_state_dict(S.make_udf_params(udf_c, 0))
    col = F.ResidualRenderingNetwork(d_feature=256, mode="no_normal", d_in=6, d_out=3, d_hidden=128, n_layers=4,
                                     weight_norm=True, multires_view=4, squeeze_out=True, blending_cand_views=10)
    col.load_state_dict(S.make_color_params(col_c, 1))
    var = F.SingleVarianceNetwork(0.6)
    beta = F.BetaNetwork(init_var_beta=0.5, init_var_gamma=0.3, init_var_zeta=0.3, beta_min=5e-5,
                         requires_grad_beta=True, requires_grad_gamma=False, requires_grad_zeta=False)
    udf, col, var, beta = [m.to(dev) for m in (udf, col, var, beta)]
    ren = UDFRendererBlending(None, udf, var, col, beta, n_samples=64, n_importance=0, n_outside=0, up_sample_steps=0,
                              perturb=0.0, h_patch_size=3)
    v = {k: x.to(dev) for k, x in S.make_blend_views(args.rays, n_views=8, seed=0).items()}
    z = (v["near"] + (v["far"] - v["near"]) * torch.linspace(0.0, 1.0, 64, device=dev)[None, :]).contiguous()
    sd = float(((v["far"] - v["near"]) / 64).mean())
    gt = loss_inputs(args.rays, 3, dev, seed=1)
    params = [p for m in (udf, col, var, beta) for p in m.parameters() if p.requires_grad]

    n = args.rays
    tex = 0.1 * (loss_inputs(n, 3, dev, seed=2)["gt_patch_colors"] - 0.5)

    def make_step(fn):
        def step():
            for p in params:
                p.grad = None
            ret = ren.render_core(v["rays_o"], v["rays_d"], z, sd, udf, var, col, beta_network=beta, cos_anneal_ratio=0.5)
            # render_core without blending has no patch colours: the patch term gets the rendered colour shifted by a
            # fixed texture, so that its gradient flows through the whole render
            patch_colors = ret["color"][:, None, :] + tex
            patch_mask = ret["weight_sum"] > 0.5
            out = fn(ret["color_base"], ret["color"], gt["gt_color"], None, gt["pixel_mask"], patch_colors,
                     gt["gt_patch_colors"], patch_mask)
            out["loss"].backward()
            return out["loss"].detach()
        return step

    def blend_forward():
        ren.render_core(v["rays_o"], v["rays_d"], z, sd, udf, var, col, beta_network=beta, cos_anneal_ratio=0.5,
                        color_maps=v["color_maps"], w2cs=v["w2cs"], intrinsics=v["intrinsics"], query_c2w=v["query_c2w"],
                        rays_uv=v["rays_uv"])

    res = {"rays": n, "samples": 64, "h": 3, "type": "ncc"}
    # the blending path of render_core (fine-tuning stage) and the torch.inverse it calls, checked for host reads
    blend_forward()
    res["blend_render_core_host_sync"] = host_sync_error(blend_forward)
    res["torch_inverse_host_sync"] = host_sync_error(lambda: torch.inverse(v["w2cs"]))
    dev_step = make_step(ColorLoss(*WEIGHTS, patch_loss_type="ncc", h_patch_size=3))
    res["eager_device_loss_ms"], _ = timed(dev_step, args.iters)
    res["eager_device_loss_kernels"], res["eager_device_loss_copies"] = count_launches(dev_step)
    res["device_loss_step_host_sync"] = host_sync_error(dev_step)
    if ref_mod is not None:
        ref_step = make_step(ref_mod.ColorLoss(*WEIGHTS, patch_loss_type="ncc", h_patch_size=3).to(dev))
        res["eager_reference_loss_ms"], _ = timed(ref_step, args.iters)
        res["eager_reference_loss_kernels"], res["eager_reference_loss_copies"] = count_launches(ref_step)
        res["reference_loss_step_host_sync"] = host_sync_error(ref_step)
    if res["device_loss_step_host_sync"] is None:
        eager_loss = dev_step().clone()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(3):
                dev_step()
        torch.cuda.current_stream().wait_stream(s)
        for p in params:
            p.grad = None
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            g_loss = dev_step()
        graph.replay()
        torch.cuda.synchronize()
        res["graph_loss_equals_eager"] = bool(torch.equal(g_loss, eager_loss))
        res["graph_replay_ms"], _ = timed(graph.replay, args.iters)
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=512)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("loss_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    ref_mod = None
    from oracle import refshim
    if refshim.available():
        from oracle.make_golden_loss import load_reference_loss
        ref_mod = load_reference_loss()
    result = {"gpu": gpu_info(), "loss": bench_loss(args, dev, ref_mod), "step": bench_step(args, dev, ref_mod),
              "gpu_after": gpu_info()}
    print(json.dumps({"gpu": result["gpu"], "gpu_after": result["gpu_after"]}))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
