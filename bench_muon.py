# -*- coding: utf-8 -*-
"""torch.optim.Muon's step on one GPU: the fused step (stk_muon_step: Newton-Schulz batched over every matrix on bf16
tensor cores, no host synchronisation) against B200StockOptimizer running the class's own step (per matrix: the
momentum lerps, then torch's bf16 matmuls / addmm on cuBLAS, five Newton-Schulz steps of three GEMMs each, the update),
on two matrix sets, with the same injected bf16 gradients, in alternating rounds in one run:

  bert      BERT-base's encoder matrices: 12 x (Q, K, V, O 768 x 768; FFN 3072 x 768 and 768 x 3072), 72 matrices,
            84.9 M elements
  resnet50  ResNet-50's 53 conv weights as (out, in kh kw) matrices, channels-last, 23.5 M elements

Both run MuonWithAuxAdamW with one Muon group (torch.optim.Muon's defaults; a conv weight is not 2-D).

  fused   CUDA events around opt.step() on the launch stream
  stock   CUDA events around opt.step() (the route reads found_inf on the host once per step)

Medians over the timed steps of every round, after a warm-up.  TFLOP/s is algorithmic: per matrix
ns_steps (4 r^2 c + 2 r^3), r <= c (X X^T: 2 r^2 c, A A: 2 r^3, B X: 2 r^2 c), over the whole step time.  The card's
name and power limit are read in the same run.

    python bench_muon.py [--out muon.json] [--iters 10] [--rounds 3] [--sets bert,resnet50]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def ns_flops(rows: int, cols: int, steps: int) -> int:
    """Algorithmic FLOPs of Newton-Schulz on one rows x cols matrix."""
    r, c = min(rows, cols), max(rows, cols)
    return steps * (4 * r * r * c + 2 * r ** 3)


def bert_base_matrices():
    """(rows, cols) of BERT-base's encoder weight matrices, as nn.Linear stores them (out, in)."""
    return [(768, 768)] * 4 * 12 + [(3072, 768), (768, 3072)] * 12


def resnet50_conv_shapes():
    """(out, in, kh, kw) of ResNet-50's conv weights in registration order (torchvision's resnet50)."""
    out = [(64, 3, 7, 7)]
    cin = 64
    for width, blocks in ((64, 3), (128, 4), (256, 6), (512, 3)):
        for b in range(blocks):
            out += [(width, cin, 1, 1), (width, width, 3, 3), (4 * width, width, 1, 1)]
            if b == 0:
                out.append((4 * width, cin, 1, 1))
            cin = 4 * width
    return out


def resnet50_matrices():
    return [(o, i * kh * kw) for o, i, kh, kw in resnet50_conv_shapes()]


def card():
    info = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_w"] = float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        pass
    return info


class Weights(torch.nn.Module):
    def __init__(self, shapes, channels_last):
        super().__init__()
        g = torch.Generator().manual_seed(0)
        self.w = torch.nn.ParameterList()
        for s in shapes:
            t = torch.randn(s, generator=g) * 0.02
            if channels_last and len(s) == 4:
                t = t.contiguous(memory_format=torch.channels_last)
            self.w.append(torch.nn.Parameter(t))


def build(shapes, channels_last, stock):
    from stoke_b200 import MuonWithAuxAdamW
    from stoke_b200.engine import get_engine
    from stoke_b200.optim import B200FusedOptimizer, B200StockOptimizer

    net = Weights(shapes, channels_last).cuda()
    kw = {"params": [dict(params=list(net.parameters()), use_muon=True)]}
    cls = B200StockOptimizer if stock else B200FusedOptimizer
    return cls(net, MuonWithAuxAdamW, kw, engine=get_engine(0), lp_dtype=torch.bfloat16)


def time_steps(opt, grads, iters):
    path = opt.path
    times = []
    for k in range(iters):
        path.g_flat.copy_(grads[k % len(grads)])
        path.after_backward(sync=True, unscale=False)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        opt.step()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sets", default="bert,resnet50")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_muon.py needs a CUDA device")
    torch.cuda.set_device(0)
    result = {"card": card(), "ns_steps": 5, "sets": {}}
    for name in args.sets.split(","):
        shapes = bert_base_matrices() if name == "bert" else resnet50_conv_shapes()
        mats = bert_base_matrices() if name == "bert" else resnet50_matrices()
        flops = sum(ns_flops(r, c, 5) for r, c in mats)
        opts = {"fused": build(shapes, name != "bert", False), "stock": build(shapes, name != "bert", True)}
        n = opts["fused"].path.n
        gen = torch.Generator(device="cuda").manual_seed(1)
        grads = [(torch.randn(n, device="cuda", generator=gen) * 1e-3).bfloat16() for _ in range(2)]
        times = {k: [] for k in opts}
        for k, opt in opts.items():
            time_steps(opt, grads, args.warmup)
        for _ in range(args.rounds):
            for k, opt in opts.items():
                times[k] += time_steps(opt, grads, args.iters)
        med = {k: statistics.median(v) for k, v in times.items()}
        result["sets"][name] = {
            "matrices": len(mats), "elements": sum(r * c for r, c in mats), "ns_gflop": flops / 1e9,
            **{f"{k}_ms": round(v, 4) for k, v in med.items()},
            **{f"{k}_tflops": round(flops / (v * 1e-3) / 1e12, 2) for k, v in med.items()},
            "speedup": round(med["stock"] / med["fused"], 2),
        }
        for opt in opts.values():
            opt.close()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
