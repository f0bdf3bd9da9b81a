# -*- coding: utf-8 -*-
"""stoke_b200.optim.LAMB and LARS on one GPU: the fused step (stk_layerwise_step, three launches, no host synchronisation)
against B200StockOptimizer running the class's own step (K1 main-gradient reduce + per-parameter torch ops on fp32 views,
two norm reductions per tensor, + the cast into the bf16 model), on the parameter sets of ResNet-50 (torchvision,
channels-last, bf16; 25.6 M elements, 161 tensors) and BERT-base (BertForSequenceClassification(BertConfig()), bf16;
109.5 M elements, 201 tensors), with the same injected gradients, in alternating rounds in one run.  One parameter group
with weight decay, so every tensor takes the trust ratio.

  fused   CUDA events around opt.step() on the launch stream (the gradient pass k_grad_norm is not in it: neither route
          needs one without clipping or a loss scaler)
  stock   a host clock around after_backward + opt.step() + torch.cuda.synchronize() (the class's step reads its step
          count on the host; the route synchronises anyway)

Medians over the timed iterations of every round, after a warm-up.  Algorithmic bytes per element on the raw bf16 route
(k2_layerwise.cu): LAMB 42 (pass 1: g, w, m, v read, m, v written, g zeroed = 24; pass 3: w, m, v read, w and the bf16
copy written = 18), LARS with momentum 28 (pass 1: g, w read = 6; pass 3: g, w, buf read, w, buf, bf16 copy written, g
zeroed = 22).  The card's name and power limit are read in the same run.

    python bench_layerwise.py [--out layerwise.json] [--iters 20] [--rounds 3] [--kinds lamb,lars]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def card():
    info = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_w"] = float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        pass
    return info


def model_of(name):
    if name == "resnet50":
        import torchvision

        return torchvision.models.resnet50().to(memory_format=torch.channels_last)
    from transformers import BertConfig, BertForSequenceClassification

    return BertForSequenceClassification(BertConfig())


BYTES_PER_ELEMENT = {"lamb": 42, "lars": 28}
KWARGS = {"lamb": {"lr": 1e-3, "weight_decay": 0.01}, "lars": {"lr": 1.0, "momentum": 0.9, "weight_decay": 5e-5}}


def run(name, kind, iters, rounds):
    from stoke_b200 import synthetic
    from stoke_b200.engine import get_engine
    from stoke_b200.optim import LAMB, LARS, B200FusedOptimizer, B200StockOptimizer

    eng = get_engine(0)
    opts = {}
    for route, cls in (("fused", B200FusedOptimizer), ("stock", B200StockOptimizer)):
        torch.manual_seed(0)
        net = model_of(name).cuda()
        opts[route] = cls(net, LAMB if kind == "lamb" else LARS, KWARGS[kind], engine=eng, lp_dtype=torch.bfloat16)
    path = opts["fused"].path
    grads = [synthetic.injected_grad(gv.numel(), 0, i, dtype=torch.bfloat16, scale=1e-3).view(gv.shape).cuda()
             for i, gv in enumerate(path.grad_views)]
    n = sum(p.numel() for p in path.params)
    nbytes = BYTES_PER_ELEMENT[kind] * n

    def fill(o):
        for gv, g in zip(o.path.grad_views, grads):
            gv.copy_(g)

    times = {"fused": [], "stock": []}
    launches = None
    for r in range(rounds + 1):   # round 0 warms up
        for route in ("fused", "stock"):
            o = opts[route]
            for _ in range(iters):
                fill(o)
                if route == "fused":
                    o.path.after_backward(sync=True, unscale=False)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    l0 = eng.launches
                    e0.record()
                    o.step()
                    e1.record()
                    e1.synchronize()
                    launches = eng.launches - l0
                    ms = e0.elapsed_time(e1)
                else:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    o.path.after_backward(sync=True, unscale=False)
                    o.step()
                    torch.cuda.synchronize()
                    ms = (time.perf_counter() - t0) * 1e3
                if r > 0:
                    times[route].append(ms)
    for o in opts.values():
        o.close()
    fused, stock = statistics.median(times["fused"]), statistics.median(times["stock"])
    return {"model": name, "optimizer": kind, "params": len(path.params), "elements": n, "algorithmic_bytes": nbytes, "fused_ms": fused, "stock_ms": stock, "speedup": stock / fused,
            "fused_tb_s": nbytes / fused / 1e9, "fused_launches": launches,
            "fused_ms_spread": [min(times["fused"]), max(times["fused"])],
            "stock_ms_spread": [min(times["stock"]), max(times["stock"])]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--models", default="resnet50,bert")
    ap.add_argument("--kinds", default="lamb,lars")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_layerwise.py needs a GPU")
    torch.cuda.set_device(0)
    res = {"card": card(), "rows": []}
    print(json.dumps({"card": res["card"]}), flush=True)
    for name in args.models.split(","):
        for kind in args.kinds.split(","):
            row = run(name, kind, args.iters, args.rounds)
            res["rows"].append(row)
            print(json.dumps(row), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
