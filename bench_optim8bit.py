# -*- coding: utf-8 -*-
"""The 8-bit optimizers of stoke_b200 on one GPU, at ResNet-50 size (25.6 M elements) and BERT-base size (109.5 M
elements), each against its fp32 kind: AdamW8bit / AdamW, Lion8bit / Lion, AdEMAMix8bit / AdEMAMix (``--kinds``):

  step[<8-bit>] vs step[<fp32>]    the fused 8-bit step (stk_adam8bit_step, stk_lion8bit_step or stk_ademamix8bit_step:
                       prologue + k_q8_step) against the fused fp32 step (k_optim_step), both on the world-1 raw bf16 route
                       with clip-by-norm, each behind its gradient pass (k_grad_norm, 2 B/element read), timed in
                       alternating rounds in the same run.  Algorithmic bytes per element of the step: AdamW 30 (read g 2,
                       p m v 12; write p m v 12, bf16 copy 2, zeroing 2), Lion 22, AdEMAMix 38; AdamW8bit 18 (read g 2,
                       master 4, codes 2; write master 4, codes 2, bf16 copy 2, zeroing 2) plus 12 B per 256 elements (two
                       absmax read and written, the block table); Lion8bit 16 (one code) plus 8 per 256; AdEMAMix8bit 20
                       (three codes) plus 24 per 256
  optimizer_step fused vs stock    the whole step (grad copy + gradient pass + step) of the 8-bit class on the fused route
                       against the same class on B200StockOptimizer (K1 main-gradient reduce + the class's own update on
                       fp32 views + the cast into the bf16 model), same gradients, alternating rounds
  kernels (torch.profiler)         per-kernel device time of a few steps of each fused route, in a separate pass

It also reports the optimizer-state bytes of both fused routes.  Timing as bench_optim.py: CUDA events on the launch
stream, medians; ResNet-50-sized rows are preceded by an L2 flush write.  The card's name and power limit are read in the
same run and printed with the numbers.

    python bench_optim8bit.py [--kinds adamw8bit,lion8bit,ademamix8bit] [--out optim8bit.json] [--iters 40] [--rounds 4]
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

# 8-bit kind -> (its fp32 kind, step bytes per element of each, the 8-bit step's bytes per 256-element block)
KINDS = {"adamw8bit": ("adamw", 18, 30, 12), "lion8bit": ("lion", 16, 22, 8), "ademamix8bit": ("ademamix", 20, 38, 24)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--iters", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--kinds", default="adamw8bit", help="comma-separated, of " + ", ".join(KINDS))
    args = ap.parse_args()
    kinds = args.kinds.split(",")
    if not set(kinds) <= set(KINDS):
        raise SystemExit(f"--kinds: each of {', '.join(KINDS)}")
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
    fp32_cls = {"adamw": torch.optim.AdamW, "lion": stoke_b200.Lion, "ademamix": stoke_b200.AdEMAMix}
    q8_cls = {"adamw8bit": stoke_b200.AdamW8bit, "lion8bit": stoke_b200.Lion8bit, "ademamix8bit": stoke_b200.AdEMAMix8bit}
    sizes = (("resnet50_25.6M", 25_557_032), ("bert_base_109.5M", 109_483_778))
    for kind, (size_name, n) in ((k, sz) for k in kinds for sz in sizes):
        ref_kind, q8_bytes, ref_bytes, block_bytes = KINDS[kind]
        classes = {kind: q8_cls[kind], ref_kind: fp32_cls[ref_kind]}
        flush_l2 = n < 60_000_000
        # ---- the fused steps, alternating ----
        opts = {k: B200FusedOptimizer(Flat(n).cuda(), cls, kw, engine=eng, route="local", clip=clip,
                                      lp_dtype=torch.bfloat16) for k, cls in classes.items()}
        grads = (torch.randn(opts[ref_kind].path.n, device="cuda") * 1e-3).to(torch.bfloat16)
        for o in opts.values():   # one real step so that the state holds non-zero moments
            o.path.g_flat.copy_(grads)
            o.path.after_backward(sync=True, unscale=False)
            o.step()
        q8, fp = opts[kind].path, opts[ref_kind].path
        state_bytes = {kind: sum(t.numel() * t.element_size() for t in (q8.q8_codes, q8.q8_code2, q8.q8_absmaxes,
                                                                         q8.q8_absmax2, q8.q8_small) if t is not None),
                       ref_kind: 4 * fp.n * sum(b is not None for b in (fp.M, fp.V, fp.M2, fp.M3))}
        nb = q8.q8_absmax1.numel()
        step_bytes = {kind: n * q8_bytes + block_bytes * nb, ref_kind: n * ref_bytes}

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
        report({"row": f"step[{kind}] / step[{ref_kind}]", "size": size_name,
                "time_ratio": med[(kind, "step")] / med[(ref_kind, "step")],
                "time_ratio_with_norm_pass": (med[(kind, "step")] + med[(kind, "norm")]) /
                                             (med[(ref_kind, "step")] + med[(ref_kind, "norm")]),
                "state_ratio": state_bytes[kind] / state_bytes[ref_kind]})
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
        del opts, q8, fp
        torch.cuda.empty_cache()
        # ---- the whole step: fused vs the stock route, alternating ----
        cls = q8_cls[kind]
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
        report({"row": f"optimizer_step[{kind}] fused vs stock (grad copy + gradient pass + step)", "size": size_name,
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
