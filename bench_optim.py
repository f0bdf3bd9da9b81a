# -*- coding: utf-8 -*-
"""torch.optim classes on the fused step, on one GPU, at ResNet-50 size (25.6 M elements) and BERT-base size
(109.5 M elements), with Adam as the yardstick.  By default Adam, NAdam, RAdam and Adamax; ``--kinds`` picks others, e.g.
``--kinds adadelta,rprop,asgd``, ``--kinds adam,lion`` (stoke_b200.Lion), ``--kinds adam,sf_adamw,sgd,sf_sgd``
(stoke_b200.AdamWScheduleFree and SGDScheduleFree against the kinds whose bytes they move), ``--kinds adam,ademamix``
(stoke_b200.AdEMAMix, Adam's step with a third state tensor), ``--kinds adam,rmsprop_tf,rmsprop_tf_centered,ademamix``
(stoke_b200.RMSpropTF with the EfficientNet recipe's settings, and centered, against the kinds whose bytes they move) or
``--kinds adam,ademamix,adan`` (stoke_b200.Adan, with a fourth state tensor):

  k_optim_step[raw]    the world-1 route: the step reads and zeroes the raw bf16 bucket and writes the bf16 model copy
                       (30 B/element algorithmic: read g 2, p m v 12; write p m v 12, bf16 copy 2, zeroing 2), with the
                       step prologue in front of it.  ASGD keeps one state tensor and, while mu == 1 (torch's default
                       t0 = 1e6), writes it without reading it: 18 B/element.  Lion keeps one state tensor, reads it
                       and runs without the prologue: 22 B/element.  SGD with momentum and schedule-free SGD keep one
                       (momentum_buffer / z): 22 B/element; schedule-free AdamW keeps two like Adam: 30.  AdEMAMix
                       keeps three (exp_avg_fast, exp_avg_slow, exp_avg_sq): 38 B/element.  RMSpropTF with momentum
                       keeps two (square_avg, momentum_buffer) and runs without the prologue: 30 B/element; centered it
                       keeps grad_avg too: 38.  Adan keeps four (exp_avg, exp_avg_sq, exp_avg_diff, neg_pre_grad): 46
  k_optim_step[main]   fp32 model, fp32 main gradients (28 B/element: read g p m v 16, write p m v 12; ASGD 16, Lion, SGD
                       and schedule-free SGD 20, AdEMAMix and centered RMSpropTF 36, Adan 44)
  optimizer step       gradient pass + step, the fused route (k_grad_norm + prologue + k_optim_step) against
                       B200StockOptimizer (K1 main-gradient reduce + the class's own update on fp32 views + the cast
                       into the bf16 model), same class, same gradients, timed in alternating rounds in the same run
  schedule-free swap   eval() + train() of the fused schedule-free optimizers on a bf16 model: per call one stk_weight_avg
                       lerp of the master toward z (read master, z; write master: 12 B/element) and the cast of the
                       master into the bf16 model (6 B/element), 36 B/element per pair

    python bench_optim.py [--out optim.json] [--iters 30] [--kinds adam,nadam,radam,adamax]

Timing as bench_kernels.py: CUDA events on the launch stream, medians; ResNet-50-sized kernel rows are preceded by an L2 flush
write.  The card's name and power limit are read in the same run and written with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import stoke_b200  # noqa: E402


def card():
    info = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_w"] = float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        pass
    return info


CLASSES = {"adam": (torch.optim.Adam, {"lr": 1e-3}), "nadam": (torch.optim.NAdam, {"lr": 2e-3}),
           "radam": (torch.optim.RAdam, {"lr": 1e-3}), "adamax": (torch.optim.Adamax, {"lr": 2e-3}),
           "adadelta": (torch.optim.Adadelta, {"lr": 1.0}), "rprop": (torch.optim.Rprop, {"lr": 1e-2}),
           "asgd": (torch.optim.ASGD, {"lr": 1e-2}), "lion": (stoke_b200.Lion, {"lr": 1e-4, "weight_decay": 0.1}),
           "sgd": (torch.optim.SGD, {"lr": 0.1, "momentum": 0.9}),
           "sf_adamw": (stoke_b200.AdamWScheduleFree, {"lr": 2.5e-3, "weight_decay": 0.01}),
           "sf_sgd": (stoke_b200.SGDScheduleFree, {"lr": 1.0, "weight_decay": 1e-4}),
           "ademamix": (stoke_b200.AdEMAMix, {"lr": 1e-3, "alpha": 5.0, "alpha_warmup": 100_000,
                                              "beta3_warmup": 100_000, "weight_decay": 0.01}),
           # timm's EfficientNet recipe (--opt rmsproptf --opt-eps .001 --momentum 0.9, weight decay 1e-5)
           "rmsprop_tf": (stoke_b200.RMSpropTF, {"lr": 0.016, "alpha": 0.9, "eps": 1e-3, "momentum": 0.9,
                                                 "weight_decay": 1e-5}),
           "rmsprop_tf_centered": (stoke_b200.RMSpropTF, {"lr": 0.016, "alpha": 0.9, "eps": 1e-3, "momentum": 0.9,
                                                          "weight_decay": 1e-5, "centered": True}),
           "adan": (stoke_b200.Adan, {"lr": 1e-3, "weight_decay": 0.02})}
# algorithmic bytes per element (raw bf16 route, main fp32 route) of the kinds with one state tensor; the others: 30, 28
ONE_STATE_BYTES = {"asgd": (18, 16),   # ax written without being read while mu == 1
                   "lion": (22, 20), "sgd": (22, 20), "sf_sgd": (22, 20)}
THREE_STATE_BYTES = {"ademamix": (38, 36),   # the first and second moments plus exp_avg_slow
                     "rmsprop_tf_centered": (38, 36),   # square_avg, momentum_buffer and grad_avg
                     "adan": (46, 44)}   # four: exp_avg, exp_avg_sq, exp_avg_diff and neg_pre_grad
SCHEDULE_FREE = ("sf_adamw", "sf_sgd")   # a new optimizer is in eval mode: train() before stepping


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--kinds", default="adam,nadam,radam,adamax",
                    help="comma-separated: " + ",".join(CLASSES))
    args = ap.parse_args()
    kinds = [k.strip() for k in args.kinds.split(",") if k.strip()]
    unknown = [k for k in kinds if k not in CLASSES]
    if unknown:
        raise SystemExit(f"bench_optim.py: unknown kinds {unknown} (known: {', '.join(CLASSES)})")
    if not torch.cuda.is_available():
        raise SystemExit("bench_optim.py needs a GPU")
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

    def report(row):
        rows.append(row)
        print(json.dumps(row), flush=True)

    class Flat(torch.nn.Module):
        def __init__(self, n):
            super().__init__()
            self.w = torch.nn.Parameter(torch.zeros(n))

    classes = [(k,) + CLASSES[k] for k in kinds]
    clip = ClipSpec(_lib.CLIP_NORM, max_norm=1.0, norm_type=2.0)
    for size_name, n in (("resnet50_25.6M", 25_557_032), ("bert_base_109.5M", 109_483_778)):
        flush_l2 = n < 60_000_000
        for tag, cls, kw in classes:
            # ---- the kernel alone, both gradient sources ----
            raw_b, main_b = ONE_STATE_BYTES.get(tag, THREE_STATE_BYTES.get(tag, (30, 28)))
            for route, lp, per in (("local", torch.bfloat16, raw_b), ("main", None, main_b)):
                net = Flat(n).cuda()
                opt = B200FusedOptimizer(net, cls, kw, engine=eng, route=route, clip=clip, lp_dtype=lp)
                if tag in SCHEDULE_FREE:
                    opt.train()
                path = opt.path
                path.g_flat.copy_((torch.randn(path.n, device="cuda") * 1e-3).to(path.g_flat.dtype))
                if route == "main":
                    path.main_flat.copy_(torch.randn(path.n, device="cuda") * 1e-3)
                step = lambda: opt.step()   # noqa: E731 -- prologue + k_optim_step + epilogue
                measure(step, 5, False)
                ms = sorted(measure(step, args.iters, flush_l2))
                med = ms[len(ms) // 2]
                nbytes = path.n * per
                report({"row": f"k_optim_step[{'raw' if route == 'local' else 'main'},{tag}] (+prologue, epilogue)",
                        "size": size_name, "us_median": med * 1e3, "us_min": ms[0] * 1e3, "bytes_per_elem": per,
                        "achieved_gbs": nbytes / (med * 1e-3) / 1e9, "frac_of_hbm_peak": nbytes / (med * 1e-3) / 1e9 / peak,
                        "l2_flush_between_launches": flush_l2})
                opt.close()
                del opt, path, net
                torch.cuda.empty_cache()
            # ---- the whole optimizer step: fused route vs the stock-optimizer route, alternating ----
            nets = {"fused": Flat(n).cuda(), "stock": Flat(n).cuda()}
            opts = {"fused": B200FusedOptimizer(nets["fused"], cls, kw, engine=eng, clip=clip, lp_dtype=torch.bfloat16),
                    "stock": B200StockOptimizer(nets["stock"], cls, kw, engine=eng, clip=clip, lp_dtype=torch.bfloat16)}
            if tag in SCHEDULE_FREE:
                for o in opts.values():
                    o.train()
            grads = (torch.randn(opts["fused"].path.n, device="cuda") * 1e-3).to(torch.bfloat16)

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
            per_round = max(1, args.iters // args.rounds)
            for _ in range(args.rounds):
                for k in ("fused", "stock"):
                    times[k] += measure(runs[k], per_round, flush_l2)
            med = {}
            for k, ms in times.items():
                ms.sort()
                med[k] = ms[len(ms) // 2]
            report({"row": f"optimizer_step[{tag}] fused vs stock (grad copy + gradient pass + step)", "size": size_name,
                    "fused_us_median": med["fused"] * 1e3, "stock_us_median": med["stock"] * 1e3,
                    "stock_over_fused": med["stock"] / med["fused"], "rounds": args.rounds,
                    "l2_flush_between_launches": flush_l2})
            if tag in SCHEDULE_FREE:
                o = opts["fused"]
                swap = lambda: (o.eval(), o.train())   # noqa: E731
                measure(swap, 3, False)
                ms = sorted(measure(swap, args.iters, flush_l2))
                nbytes = o.path.n * 36
                report({"row": f"schedule_free_swap[{tag}] eval() + train(), bf16 model", "size": size_name,
                        "us_median": ms[len(ms) // 2] * 1e3, "us_min": ms[0] * 1e3, "bytes_per_elem": 36,
                        "achieved_gbs": nbytes / (ms[len(ms) // 2] * 1e-3) / 1e9, "l2_flush_between_launches": flush_l2})
            for o in opts.values():
                o.close()
            del opts, nets, runs
            torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": gpu, "peak_hbm_gbs": peak, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
