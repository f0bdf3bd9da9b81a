# -*- coding: utf-8 -*-
"""bench_bn_stats.py -- the BatchNorm forward of every fused ResNet-50 site at B = 128, two ways (CUDA events over
back-to-back calls after warm-up, bf16 channels-last, fp32 running statistics):

  torch + apply   torch.batch_norm_update_stats (semaphore fill, statistics, running-statistics update) + stk_bn_act_ex
  fused           stk_bn_stats_act: the same results in one cooperative launch

and torch's statistics alone.  Bytes counted: 2 B/element for the statistics, 4 (6 with the residual) for the apply.
Prints one JSON line per site shape, then the step totals weighted by the number of sites of each shape, with the GPU's
name and power limit.

    python bench_bn_stats.py [--iters N] [--batch B]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

# (C, H = W, residual, sites) of the 49 fused BatchNorms of torchvision's ResNet-50
SITES = [(64, 112, False, 1), (64, 56, False, 6), (256, 56, True, 3), (128, 56, False, 1), (128, 28, False, 7),
         (512, 28, True, 4), (256, 28, False, 1), (256, 14, False, 11), (1024, 14, True, 6), (512, 14, False, 1),
         (512, 7, False, 5), (2048, 7, True, 3)]


def _time(fn, iters, torch):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--batch", type=int, default=128)
    args = ap.parse_args()
    import torch

    from stoke_b200._lib import ACT_RELU
    from stoke_b200.engine import get_engine

    if not torch.cuda.is_available():
        raise SystemExit("bench_bn_stats.py needs a CUDA device")
    torch.cuda.set_device(0)
    eng = get_engine(0)
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    assert sum(s[3] for s in SITES) == 49
    tot = {"torch_us": 0.0, "torch_stats_us": 0.0, "fused_us": 0.0}
    for c, hw, res, sites in SITES:
        g = torch.Generator(device="cuda").manual_seed(c + hw)
        shape = (args.batch, c, hw, hw)
        x = torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        r = torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=torch.channels_last) if res else None
        w = torch.rand(c, device="cuda", generator=g).to(torch.bfloat16) + 0.5
        b = torch.rand(c, device="cuda", generator=g).to(torch.bfloat16) - 0.5
        rm, rv = torch.zeros(c, device="cuda"), torch.ones(c, device="cuda")
        out, mean, inv = torch.empty_like(x), torch.empty(c, device="cuda"), torch.empty(c, device="cuda")

        def unfused():
            m, v = torch.batch_norm_update_stats(x, rm, rv, 0.1)
            eng.bn_act(x, r, m, v, w, b, 1e-5, out, inv, ACT_RELU)

        def stats():
            torch.batch_norm_update_stats(x, rm, rv, 0.1)

        def fused():
            eng.bn_stats_act(x, r, w, b, rm, rv, 0.1, 1e-5, out, mean, inv, ACT_RELU)

        t_unf, t_st, t_fus = (_time(f, args.iters, torch) for f in (unfused, stats, fused))
        n = x.numel()
        apply_b = n * (6 if res else 4)
        row = {"C": c, "HW": hw, "residual": res, "sites": sites, "torch_us": round(t_unf, 1),
               "torch_stats_us": round(t_st, 1), "fused_us": round(t_fus, 1), "speedup": round(t_unf / t_fus, 2),
               "torch_stats_TBps": round(2 * n / t_st / 1e6, 2), "fused_TBps": round((2 * n + apply_b) / t_fus / 1e6, 2)}
        print(json.dumps(row))
        tot["torch_us"] += sites * t_unf
        tot["torch_stats_us"] += sites * t_st
        tot["fused_us"] += sites * t_fus
        del x, r, out
    print(json.dumps({"gpu": gpu, "batch": args.batch, "sites": 49, **{k: round(v, 1) for k, v in tot.items()},
                      "saved_us_per_step": round(tot["torch_us"] - tot["fused_us"], 1)}))


if __name__ == "__main__":
    main()
