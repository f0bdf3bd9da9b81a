# -*- coding: utf-8 -*-
"""stoke_b200.AdamW8bit on one GPU, at ResNet-50 size (25.6 M elements) and BERT-base size (109.5 M elements):

  step[adamw8bit] vs step[adamw]   the fused 8-bit step (stk_adam8bit_step: prologue + k_q8_step) against the fused
                       AdamW step (k_optim_step), both on the world-1 raw bf16 route with clip-by-norm, each behind its
                       gradient pass (k_grad_norm, 2 B/element read), timed in alternating rounds in the same run.
                       Algorithmic bytes per element of the step: AdamW 30 (read g 2, p m v 12; write p m v 12, bf16 copy
                       2, zeroing 2); AdamW8bit 18 (read g 2, master 4, codes 2; write master 4, codes 2, bf16 copy 2,
                       zeroing 2) plus 12 B per 256 elements (two absmax read and written, the block table)
  optimizer_step fused vs stock    the whole step (grad copy + gradient pass + step) of AdamW8bit on the fused route
                       against the same class on B200StockOptimizer (K1 main-gradient reduce + the class's own update on
                       fp32 views + the cast into the bf16 model), same gradients, alternating rounds
  kernels (torch.profiler)         per-kernel device time of a few steps of each fused route, in a separate pass

It also reports the optimizer-state bytes of both fused routes.  Timing as bench_optim.py: CUDA events on the launch
stream, medians; ResNet-50-sized rows are preceded by an L2 flush write.  The card's name and power limit are read in the
same run and printed with the numbers.

    python bench_optim8bit.py [--out optim8bit.json] [--iters 40] [--rounds 4]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import stoke_b200  # noqa: E402
from bench_optim import card  # noqa: E402

Q8_BYTES, ADAMW_BYTES = 18, 30


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--iters", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=4)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_optim8bit.py needs a GPU")
    from stoke_b200 import _lib
    from stoke_b200.engine import ClipSpec, get_engine
    from stoke_b200.optim import B200FusedOptimizer, B200StockOptimizer

    torch.cuda.set_device(0)
    eng = get_engine(0)
    peak = 3350.0   # H100 SXM data sheet, HBM3
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    rows = []
    gpu = card()
    print(json.dumps({"card": gpu}), flush=True)

    def measure(fn, iters, flush_l2):
        ms = []
        for _ in range(iters):
            if flush_l2:
                flush.fill_(1)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        return ms

    def median(ms):
        return sorted(ms)[len(ms) // 2]

    def report(row):
        rows.append(row)
        print(json.dumps(row), flush=True)

    class Flat(torch.nn.Module):
        def __init__(self, n):
            super().__init__()
            self.w = torch.nn.Parameter(torch.zeros(n))

    clip = ClipSpec(_lib.CLIP_NORM, max_norm=1.0, norm_type=2.0)
    kw = {"lr": 1e-3, "weight_decay": 0.01}
    classes = {"adamw8bit": stoke_b200.AdamW8bit, "adamw": torch.optim.AdamW}
    for size_name, n in (("resnet50_25.6M", 25_557_032), ("bert_base_109.5M", 109_483_778)):
        flush_l2 = n < 60_000_000
        # ---- the fused steps, alternating ----
        opts = {k: B200FusedOptimizer(Flat(n).cuda(), cls, kw, engine=eng, route="local", clip=clip,
                                      lp_dtype=torch.bfloat16) for k, cls in classes.items()}
        grads = (torch.randn(opts["adamw"].path.n, device="cuda") * 1e-3).to(torch.bfloat16)
        for o in opts.values():   # one real step so that the state holds non-zero moments
            o.path.g_flat.copy_(grads)
            o.path.after_backward(sync=True, unscale=False)
            o.step()
        q8 = opts["adamw8bit"].path
        state_bytes = {"adamw8bit": 2 * q8.q8_code1.numel() + 8 * q8.q8_absmax1.numel() + 4 * q8.q8_small.numel(),
                       "adamw": 8 * opts["adamw"].path.n}
        nb = q8.q8_absmax1.numel()
        step_bytes = {"adamw8bit": n * Q8_BYTES + 12 * nb, "adamw": n * ADAMW_BYTES}

        def norm_pass(o):
            return lambda: o.path.after_backward(sync=True, unscale=False)   # k_grad_norm over the bucket

        times = {(k, part): [] for k in opts for part in ("norm", "step")}
        for k, o in opts.items():
            measure(norm_pass(o), 3, False)
            measure(o.step, 3, False)
        per_round = max(1, args.iters // args.rounds)
        for _ in range(args.rounds):
            for k, o in opts.items():
                for _ in range(per_round):
                    times[(k, "norm")] += measure(norm_pass(o), 1, flush_l2)
                    times[(k, "step")] += measure(o.step, 1, flush_l2)
        med = {key: median(ms) for key, ms in times.items()}
        for k in opts:
            report({"row": f"step[{k}] raw bf16 route, clip by norm", "size": size_name,
                    "k_grad_norm_us_median": med[(k, "norm")] * 1e3,
                    "step_us_median": med[(k, "step")] * 1e3, "step_bytes_per_elem": step_bytes[k] / n,
                    "step_achieved_gbs": step_bytes[k] / (med[(k, "step")] * 1e-3) / 1e9,
                    "step_frac_of_hbm_peak": step_bytes[k] / (med[(k, "step")] * 1e-3) / 1e9 / peak,
                    "k_grad_norm_achieved_gbs": 2 * n / (med[(k, "norm")] * 1e-3) / 1e9,
                    "optimizer_state_bytes": state_bytes[k], "state_bytes_per_elem": state_bytes[k] / n,
                    "rounds": args.rounds, "l2_flush_between_launches": flush_l2})
        report({"row": "step[adamw8bit] / step[adamw]", "size": size_name,
                "time_ratio": med[("adamw8bit", "step")] / med[("adamw", "step")],
                "time_ratio_with_norm_pass": (med[("adamw8bit", "step")] + med[("adamw8bit", "norm")]) /
                                             (med[("adamw", "step")] + med[("adamw", "norm")]),
                "state_ratio": state_bytes["adamw8bit"] / state_bytes["adamw"]})
        # ---- where the time goes: per-kernel device time, profiler on, in a pass of its own ----
        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for o in opts.values():
                for _ in range(5):
                    o.path.after_backward(sync=True, unscale=False)
                    o.step()
            torch.cuda.synchronize()
        kernels = {}
        for ev in prof.key_averages():
            if ev.device_type == torch.autograd.DeviceType.CUDA and ev.count:
                kernels[ev.key[:80]] = {"calls": ev.count, "us_per_call": ev.device_time_total / ev.count}
        report({"row": "kernels (torch.profiler, 5 steps of each route)", "size": size_name, "kernels": kernels})
        for o in opts.values():
            o.close()
        del opts, q8
        torch.cuda.empty_cache()
        # ---- the whole step: fused vs the stock route, alternating ----
        cls = stoke_b200.AdamW8bit
        opts = {"fused": B200FusedOptimizer(Flat(n).cuda(), cls, kw, engine=eng, clip=clip, lp_dtype=torch.bfloat16),
                "stock": B200StockOptimizer(Flat(n).cuda(), cls, kw, engine=eng, clip=clip, lp_dtype=torch.bfloat16)}

        def whole(o):
            def run():
                o.path.g_flat.copy_(grads)   # the same gradients into each route's bucket (2 B/elem, both routes)
                o.path.after_backward(sync=True, unscale=False)
                o.step()
            return run

        runs = {k: whole(o) for k, o in opts.items()}
        for k in runs:
            measure(runs[k], 3, False)
        times = {"fused": [], "stock": []}
        for _ in range(args.rounds):
            for k in ("fused", "stock"):
                times[k] += measure(runs[k], per_round, flush_l2)
        med = {k: median(ms) for k, ms in times.items()}
        report({"row": "optimizer_step[adamw8bit] fused vs stock (grad copy + gradient pass + step)", "size": size_name,
                "fused_us_median": med["fused"] * 1e3, "stock_us_median": med["stock"] * 1e3,
                "stock_over_fused": med["stock"] / med["fused"], "rounds": args.rounds,
                "l2_flush_between_launches": flush_l2})
        for o in opts.values():
            o.close()
        del opts, runs, grads
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": gpu, "peak_hbm_gbs": peak, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
