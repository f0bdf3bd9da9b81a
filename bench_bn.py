# -*- coding: utf-8 -*-
"""Backward of the fused BatchNorm -> [add] -> ReLU sites of ResNet-50 (bf16, channels-last, B = 128) on one GPU.

  per shape   torch's backward chain (threshold_backward + native_batch_norm_backward, what autograd runs for the unfused
              ops) against stk_bn_act_backward, with and without the residual add.  Algorithmic bytes per element: torch
              16 (threshold 6, reduce 4, elementwise 6); fused 10 without the residual (reduce 4, elementwise 6), 14 with
              it (reduce 8, elementwise 6).  The per-step total weights each shape by its number of sites.
  --profile   a torch.profiler trace of ResNet-50 forward + backward steps (the fused model, no optimizer), run apart from
              the timing: device time per step of threshold_backward, torch's BatchNorm backward reduce and elementwise
              kernels, and the engine's backward kernels.

    python bench_bn.py [--iters 50] [--profile] [--out bn.json]

Timing: CUDA events around `iters` back-to-back calls after warm-up.  Where the engine has no backward entry point,
only torch's chain is timed.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

B = 128
EPS = 1e-5


def resnet50_sites():
    """{(C, H, residual): number of fused sites} of torchvision's ResNet-50 at 224 x 224 (the stem, then per bottleneck
    BN1 -> ReLU, BN2 -> ReLU, BN3 -> add -> ReLU; the downsample BatchNorms are not fused)."""
    sites = {(64, 112, False): 1}
    for width, blocks, h_in, h_out in [(64, 3, 56, 56), (128, 4, 56, 28), (256, 6, 28, 14), (512, 3, 14, 7)]:
        for i in range(blocks):
            for key in [(width, h_in if i == 0 else h_out, False), (width, h_out, False), (4 * width, h_out, True)]:
                sites[key] = sites.get(key, 0) + 1
    return sites


def timed(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters   # us per call


def bench_shapes(eng, iters):
    fused_ok = hasattr(eng, "bn_act_backward")
    rows, tot_torch, tot_fused = [], 0.0, 0.0
    for (c, h, res), count in sorted(resnet50_sites().items()):
        shape = (B, c, h, h)
        cl = torch.channels_last
        g = torch.Generator(device="cuda").manual_seed(c + h)
        x = torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=cl)
        r = torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=cl)
        gy = torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=cl)
        w = (torch.rand(c, device="cuda") + 0.5).to(torch.bfloat16)
        b = (torch.rand(c, device="cuda") - 0.5).to(torch.bfloat16)
        rm, rv = torch.zeros(c, device="cuda"), torch.ones(c, device="cuda")
        mean, var = torch.batch_norm_update_stats(x, rm, rv, 0.1)
        out, invstd = torch.empty_like(x), torch.empty_like(mean)
        eng.bn_act(x, r if res else None, mean, var, w, b, EPS, out, invstd)

        def torch_chain():
            gg = torch.ops.aten.threshold_backward(gy, out, 0)
            torch.ops.aten.native_batch_norm_backward(gg, x, w, rm, rv, mean, invstd, True, EPS, [True, True, True])

        n = x.numel()
        row = {"C": c, "H": h, "residual": res, "sites": count, "elements": n,
               "torch_us": timed(torch_chain, iters)}
        row["torch_gbs"] = 16 * n / row["torch_us"] / 1e3
        tot_torch += count * row["torch_us"]
        if fused_ok:
            dx, dw, db = torch.empty_like(x), torch.empty_like(w), torch.empty_like(w)
            dr = torch.empty_like(x) if res else None

            def fused():
                eng.bn_act_backward(gy, x, out if res else None, mean, invstd, w, None if res else b, dx, dw, db, dr)

            row["fused_us"] = timed(fused, iters)
            row["fused_gbs"] = (14 if res else 10) * n / row["fused_us"] / 1e3
            row["speedup"] = row["torch_us"] / row["fused_us"]
            tot_fused += count * row["fused_us"]
        rows.append(row)
        print(json.dumps({k: round(v, 2) if isinstance(v, float) else v for k, v in row.items()}), flush=True)
        del x, r, gy, out
    total = {"per_step_torch_ms": tot_torch / 1e3}
    if fused_ok:
        total["per_step_fused_ms"] = tot_fused / 1e3
    print(json.dumps(total), flush=True)
    return rows, total


def profile_step(eng, steps=3):
    from torch.profiler import ProfilerActivity, profile

    from stoke_b200 import synthetic
    from stoke_b200.fuse import fuse_bn_act

    model = synthetic.resnet50().to(device="cuda", dtype=torch.bfloat16, memory_format=torch.channels_last)
    fwd = fuse_bn_act(model, eng)
    assert fwd is not None, "ResNet-50 has no fusable site"
    x, y = synthetic.resnet50_batch(B)
    x = x.to(device="cuda", dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    y = y.cuda()
    lossf = torch.nn.CrossEntropyLoss()

    def step():
        model.zero_grad(set_to_none=True)
        lossf(fwd(x).float(), y).backward()

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            step()
        torch.cuda.synchronize()
    cats = {"threshold_backward": ("threshold",), "bn_backward_reduce (torch)": ("batch_norm_backward_reduce",),
            "bn_backward_elemt (torch)": ("batch_norm_backward_elemt",), "k_bn_bwd (engine)": ("k_bn_bwd",),
            "k_bn_act (engine)": ("k_bn_act",)}
    out = {k: {"ms_per_step": 0.0, "launches_per_step": 0} for k in cats}
    for ev in prof.key_averages():
        for k, keys in cats.items():
            if any(s in ev.key for s in keys):
                out[k]["ms_per_step"] += ev.device_time_total / 1e3 / steps
                out[k]["launches_per_step"] += ev.count // steps
    for v in out.values():
        v["ms_per_step"] = round(v["ms_per_step"], 3)
    print(json.dumps({"profile": out}), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from stoke_b200.engine import get_engine

    torch.cuda.set_device(0)
    eng = get_engine(0)
    props = torch.cuda.get_device_properties(0)
    result = {"gpu": props.name}
    result["rows"], result["total"] = bench_shapes(eng, max(50, args.iters))
    if args.profile:
        result["profile"] = profile_step(eng)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
