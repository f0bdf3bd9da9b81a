# -*- coding: utf-8 -*-
"""The weight-average update (EMA / SWA, WeightAverageConfig) on one GPU, in two parts.

Kernels: the fused Adam step on the raw bf16 route (B200FusedOptimizer.step: K2 plus its one-thread epilogue) over the
parameter sets of ResNet-50 (torchvision, channels-last; 25,557,040 flat elements) and BERT-base
(BertForSequenceClassification(BertConfig()); 109,483,792), three ways:

  k2          the step alone                                                   30 B/element
  k2_then_wa  the step, then stk_weight_avg over the fp32 master: what a due   42 B/element (two launches)
              update costs on the engine
  k2_then_fe  the step, then torch._foreach_lerp_ over per-parameter fp32 views of the master: the best a user with
              access to the master could write                                 42 B/element

A fourth form, the lerp carried inside K2's own pass (38 B/element), was measured slower than k2_then_wa and is not
part of the engine (DESIGN.md section 4).

Each is timed with CUDA events around ``--iters`` back-to-back steps after a warm-up, in alternating rounds; the median
round is reported, with the algorithmic bytes over that time as TB/s.

End to end: ``Stoke`` on ResNet-50 (B = 128, bf16 channels-last, Adam, clip by norm 1.0), averaging every step against
not configured, alternated, ``--runs`` runs each: ms per step from a host clock around ``--steps`` steps ending in a
device synchronise.  The card's name and power limit are read in the same run.

    python bench_weight_avg.py [--out weight_avg.json] [--iters 50] [--rounds 3] [--runs 3] [--steps 30]
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

BYTES_PER_ELEMENT = {"k2": 30, "k2_then_wa": 42, "k2_then_fe": 42}
ADAM = {"lr": 1e-3, "betas": (0.9, 0.999), "eps": 1e-8}


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


def kernels(name, iters, rounds):
    from stoke_b200.engine import get_engine
    from stoke_b200.optim import B200FusedOptimizer
    from stoke_b200.weight_average import LERP

    torch.cuda.set_device(0)
    model = model_of(name).cuda()
    opt = B200FusedOptimizer(model, torch.optim.Adam, ADAM, engine=get_engine(0), lp_dtype=torch.bfloat16)
    path = opt.path
    assert path.route == "local"
    path.enable_weight_average()
    w = 1e-3
    avg_views, master_views = path.unflatten(path.avg_flat), path.unflatten(path.master_flat)

    def k2():
        opt.step()

    def k2_then_wa():
        path.avg_due = (LERP, w)   # what Stoke.step hands a step with an update due
        opt.step()

    def k2_then_fe():
        opt.step()
        torch._foreach_lerp_(avg_views, master_views, w)

    cases = {"k2": k2, "k2_then_wa": k2_then_wa, "k2_then_fe": k2_then_fe}
    times = {c: [] for c in cases}
    for fn in cases.values():
        for _ in range(5):
            fn()
    torch.cuda.synchronize()
    for _ in range(rounds):
        for c, fn in cases.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                fn()
            e1.record()
            e1.synchronize()
            times[c].append(e0.elapsed_time(e1) * 1e3 / iters)
    n = path.n
    out = {"n": n, "tensors": len(path.params)}
    for c in cases:
        us = statistics.median(times[c])
        out[c] = {"us": round(us, 1), "us_rounds": [round(t, 1) for t in times[c]], "bytes_per_element": BYTES_PER_ELEMENT[c],
                  "tb_per_s": round(BYTES_PER_ELEMENT[c] * n / (us * 1e-6) / 1e12, 3)}
    opt.close()
    del model, opt
    torch.cuda.empty_cache()
    return out


def end_to_end(runs, steps, warmup=5, batch=128):
    import stoke_b200 as sb
    from stoke_b200 import synthetic

    x, y = synthetic.resnet50_batch(batch)
    x, y = x.contiguous(memory_format=torch.channels_last).cuda(), y.cuda()
    res = {"off": [], "ema_every_step": []}
    for _ in range(runs):
        for arm in res:
            cfg = [sb.WeightAverageConfig(decay=0.9999)] if arm != "off" else None
            model = synthetic.resnet50().to(memory_format=torch.channels_last)
            s = sb.Stoke(model=model, optimizer=sb.StokeOptimizer(optimizer=torch.optim.Adam, optimizer_kwargs=ADAM),
                         loss=torch.nn.CrossEntropyLoss(), batch_size_per_device=batch, gpu=True, fp16="bf16",
                         grad_clip=sb.ClipGradNormConfig(max_norm=1.0, norm_type=2.0), configs=cfg, verbose=False)
            for _ in range(warmup):
                s.backward(s.loss(s.model(x), y))
                s.step()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(steps):
                s.backward(s.loss(s.model(x), y))
                s.step()
            torch.cuda.synchronize()
            res[arm].append(round((time.perf_counter() - t0) * 1e3 / steps, 3))
            if cfg is not None:
                assert s.weight_average.n_averaged == warmup + steps
            s.close()
            del s, model
            torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--workloads", default="resnet50,bert")
    ap.add_argument("--no-e2e", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_weight_avg.py needs a CUDA device")
    res = {"card": card(), "kernels": {}}
    for name in args.workloads.split(","):
        res["kernels"][name] = kernels(name, args.iters, args.rounds)
        print(name, json.dumps(res["kernels"][name]), flush=True)
    if not args.no_e2e:
        res["resnet50_e2e_ms_per_step"] = end_to_end(args.runs, args.steps)
        print("e2e", json.dumps(res["resnet50_e2e_ms_per_step"]), flush=True)
    res["card_after"] = card()
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
