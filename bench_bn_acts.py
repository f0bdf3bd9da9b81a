# -*- coding: utf-8 -*-
"""The fused BatchNorm -> SiLU / Hardswish / ReLU6 (and ReLU) sites of EfficientNet-B0 and MobileNetV3-Large on one GPU
(bf16, channels-last, training mode, B = 128, 224 x 224).

  per shape   one site's forward + backward: torch's unfused chain (native_batch_norm, the activation, its backward op,
              native_batch_norm_backward: what autograd runs for BatchNorm2d -> act) against the fused one
              (batch_norm_update_stats, stk_bn_act_ex, stk_bn_act_backward_ex).  Algorithmic bytes per element beyond
              the statistics pass both share: torch 8 forward (apply 4, activation 4) + 16 backward (activation 6,
              reduce 4, elementwise 6); fused 4 + 10.  The per-model total weights each shape by its number of sites.
  model       a whole forward + backward of the model (no optimizer) with and without the fuse_bn_act rewrite, runs
              alternated in one process.

    python bench_bn_acts.py [--models efficientnet_b0,mobilenet_v3_large] [--iters 30] [--rounds 3] [--steps 10]
                            [--out result.json]

The site shapes are found by running each model once on the meta device with forward hooks on the rewritten graph's
BnAct modules (``stoke_b200.fuse.site_shapes``).  Timing: CUDA events around back-to-back calls after warm-up.  Prints
one JSON line per row; --out also writes the whole result (to a path outside the source tree)."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

B, HW = 128, 224
MODELS = ("efficientnet_b0", "mobilenet_v3_large")


def site_shapes(name, hw=HW):
    """{(act, C, H, W, eps, momentum): number of sites} of torchvision's ``name`` after fuse_bn_act, from one forward
    of the rewritten graph on the meta device (no arithmetic)."""
    import torchvision

    from stoke_b200.fuse import fuse_bn_act, site_shapes as fused_site_shapes

    with torch.device("meta"):
        fwd = fuse_bn_act(getattr(torchvision.models, name)(), None)
        return fused_site_shapes(fwd, torch.empty(2, 3, hw, hw))


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


def bench_site(eng, act, c, h, w, eps, momentum, iters):
    from stoke_b200.fuse import _ACT_BACKWARD, _DEFAULT_ACT_FN

    shape, cl = (B, c, h, w), torch.channels_last
    g = torch.Generator(device="cuda").manual_seed(c + h)
    x = torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=cl)
    gy = torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=cl)
    wt = (torch.rand(c, device="cuda") + 0.5).to(torch.bfloat16)
    b = (torch.rand(c, device="cuda") - 0.5).to(torch.bfloat16)
    rm, rv = torch.zeros(c, device="cuda"), torch.ones(c, device="cuda")
    act_fn, act_bwd = _DEFAULT_ACT_FN[act], _ACT_BACKWARD[act]

    def torch_chain():
        y, mean, invstd = torch.ops.aten.native_batch_norm(x, wt, b, rm, rv, True, momentum, eps)
        act_fn(y)
        gg = act_bwd(gy, y)
        torch.ops.aten.native_batch_norm_backward(gg, x, wt, rm, rv, mean, invstd, True, eps, [True, True, True])

    out, dx, dw, db = torch.empty_like(x), torch.empty_like(x), torch.empty_like(wt), torch.empty_like(wt)

    def fused():
        mean, var = torch.batch_norm_update_stats(x, rm, rv, momentum)
        invstd = torch.empty_like(mean)
        eng.bn_act(x, None, mean, var, wt, b, eps, out, invstd, act)
        eng.bn_act_backward(gy, x, None, mean, invstd, wt, b, dx, dw, db, None, act)

    def stats():
        torch.batch_norm_update_stats(x, rm, rv, momentum)

    n = x.numel()
    row = {"act": ["relu", "silu", "hardswish", "relu6"][act], "C": c, "H": h, "W": w, "elements": n,
           "torch_us": timed(torch_chain, iters), "fused_us": timed(fused, iters), "stats_us": timed(stats, iters)}
    # bytes beyond the shared statistics pass, over the time beyond it
    row["torch_tbs"] = 24 * n / max(row["torch_us"] - row["stats_us"], 1e-3) / 1e6
    row["fused_tbs"] = 14 * n / max(row["fused_us"] - row["stats_us"], 1e-3) / 1e6
    row["speedup"] = row["torch_us"] / row["fused_us"]
    return row


def bench_shapes(eng, name, iters):
    rows, tot_torch, tot_fused = [], 0.0, 0.0
    for (act, c, h, w, eps, momentum), count in sorted(site_shapes(name).items()):
        row = bench_site(eng, act, c, h, w, eps, momentum, iters)
        row.update(model=name, sites=count)
        tot_torch += count * row["torch_us"]
        tot_fused += count * row["fused_us"]
        rows.append(row)
        print(json.dumps({k: round(v, 3) if isinstance(v, float) else v for k, v in row.items()}), flush=True)
        torch.cuda.empty_cache()
    total = {"model": name, "sites_torch_ms": tot_torch / 1e3, "sites_fused_ms": tot_fused / 1e3}
    print(json.dumps(total), flush=True)
    return rows, total


def bench_model(eng, name, rounds, steps):
    """Whole forward + backward per step, rewritten and not, alternated: rounds x (unfused, fused), each `steps` steps."""
    import torchvision

    from stoke_b200.fuse import fuse_bn_act

    torch.manual_seed(0)
    model = getattr(torchvision.models, name)().to(device="cuda", dtype=torch.bfloat16, memory_format=torch.channels_last)
    fwd = fuse_bn_act(model, eng)
    assert fwd is not None
    x = torch.randn(B, 3, HW, HW, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (B,), device="cuda")
    lossf = torch.nn.CrossEntropyLoss()
    arms = {"unfused": model, "fused": fwd}

    def step(f):
        model.zero_grad(set_to_none=True)
        lossf(f(x).float(), y).backward()

    for f in arms.values():
        for _ in range(3):
            step(f)
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for k, f in arms.items():
            times[k].append(timed(lambda: step(f), steps) / 1e3)   # ms per step
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    res = {"model": name, "step_ms": times, "median_ms": med, "saved_ms": med["unfused"] - med["fused"],
           "fused_sites": fwd.fused_sites}
    print(json.dumps(res), flush=True)
    return res


def gpu_conditions():
    props = torch.cuda.get_device_properties(0)
    info = {"gpu": props.name}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit,sm_clock,max_sm_clock"] = q
    except (OSError, subprocess.SubprocessError):
        info["power_limit,sm_clock,max_sm_clock"] = "unavailable"
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default=",".join(MODELS))
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_bn_acts.py measures on a GPU; none is visible")
    from stoke_b200.engine import get_engine

    torch.cuda.set_device(0)
    eng = get_engine(0)
    result = {"conditions": gpu_conditions(), "shapes": {}, "models": {}}
    print(json.dumps(result["conditions"]), flush=True)
    for name in args.models.split(","):
        result["shapes"][name] = bench_shapes(eng, name, args.iters)
    for name in args.models.split(","):
        result["models"][name] = bench_model(eng, name, args.rounds, args.steps)
    result["conditions_after"] = gpu_conditions()
    print(json.dumps(result["conditions_after"]), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
