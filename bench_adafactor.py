# -*- coding: utf-8 -*-
"""torch.optim.Adafactor on one GPU: the fused step (stk_adafactor_step, eight launches, no host synchronisation) against
B200StockOptimizer (K1 main-gradient reduce + torch's own _single_tensor_adafactor on fp32 views, two .item() per
parameter, + the cast into the bf16 model), on the parameter sets of ResNet-50 (torchvision, channels-last, bf16) and
BERT-base (BertForSequenceClassification(BertConfig()), bf16), with the same injected gradients, in alternating rounds in
one run.

  fused   CUDA events around opt.step() on the launch stream (the gradient pass k_grad_norm is not in it: neither route
          needs one without clipping or a loss scaler)
  stock   a host clock around after_backward + opt.step() + torch.cuda.synchronize() (the route synchronises anyway)

Medians over the timed iterations of every round, after a warm-up.  Algorithmic bytes come from the shapes (raw bf16
route): g 2 B per read (4 reads for a factored parameter: row sums, column sums, ||u||, update; 2 for a vector), w 4 B x 2
reads + 4 B write, bf16 copy 2 B, bucket zeroing 2 B, plus the state (factored: row_var / col_var read + written by the
lerp and read again by the row means, ||u|| and the update, counted as 5 x 4 B per state element; vectors: variance read +
written, read again: 12 B per element).  The card's name and power limit are read in the same run.

    python bench_adafactor.py [--out adafactor.json] [--iters 20] [--rounds 3]
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


def algorithmic_bytes(params):
    from stoke_b200 import layout

    n = nbytes = nstate = 0
    for p in params:
        lay = layout.adafactor_layout(p.shape, p.stride())
        k, s = lay["numel"], lay["state"]
        n, nstate = n + k, nstate + s
        nbytes += (2 * 4 + 12 + 4) * k + 20 * s if lay["factored"] else (2 * 2 + 12 + 4) * k + 12 * s
    return n, nbytes, nstate


def run(name, iters, rounds, kw):
    from stoke_b200 import synthetic
    from stoke_b200.engine import get_engine
    from stoke_b200.optim import B200FusedOptimizer, B200StockOptimizer

    eng = get_engine(0)
    opts = {}
    for kind, cls in (("fused", B200FusedOptimizer), ("stock", B200StockOptimizer)):
        torch.manual_seed(0)
        net = model_of(name).cuda()
        opts[kind] = cls(net, torch.optim.Adafactor, kw, engine=eng, lp_dtype=torch.bfloat16)
    path = opts["fused"].path
    grads = [synthetic.injected_grad(gv.numel(), 0, i, dtype=torch.bfloat16, scale=1e-3).view(gv.shape).cuda()
             for i, gv in enumerate(path.grad_views)]
    n, nbytes, nstate = algorithmic_bytes(path.params)

    def fill(o):
        for gv, g in zip(o.path.grad_views, grads):
            gv.copy_(g)

    times = {"fused": [], "stock": []}
    launches = None
    for r in range(rounds + 1):   # round 0 warms up
        for kind in ("fused", "stock"):
            o = opts[kind]
            for _ in range(iters):
                fill(o)
                if kind == "fused":
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
                    times[kind].append(ms)
    for o in opts.values():
        o.close()
    fused, stock = statistics.median(times["fused"]), statistics.median(times["stock"])
    return {"model": name, "params": len(path.params), "elements": n, "state_elements": nstate,
            "algorithmic_bytes": nbytes, "fused_ms": fused, "stock_ms": stock, "speedup": stock / fused,
            "fused_tb_s": nbytes / fused / 1e9, "fused_launches": launches,
            "fused_ms_spread": [min(times["fused"]), max(times["fused"])],
            "stock_ms_spread": [min(times["stock"]), max(times["stock"])]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--models", default="resnet50,bert")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_adafactor.py needs a GPU")
    torch.cuda.set_device(0)
    res = {"card": card(), "rows": []}
    print(json.dumps({"card": res["card"]}), flush=True)
    for name in args.models.split(","):
        row = run(name, args.iters, args.rounds, {"lr": 1e-2})
        res["rows"].append(row)
        print(json.dumps(row), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
