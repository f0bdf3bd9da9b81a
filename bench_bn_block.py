# -*- coding: utf-8 -*-
"""bench_bn_block.py -- ResNet-50's block boundary at B = 128 (bf16 channels-last).  First the forward of the 4
downsample sites: torch's BatchNorm on the residual followed by the residual site, against the two-BatchNorm site
(stk_bn_stats_act with weight2).  Then the backward of the forked block outputs, two ways:

  add + site   autograd's bf16 add of the output's two gradients, then stk_bn_act_backward_ex at the residual site
  forked       stk_bn_act_backward_ex with the second gradient (grad2): the sum is formed inside the reduce kernel

timed with CUDA events over back-to-back calls after warm-up.  Bytes per element from shapes: the add reads 4 and writes
2; the site's reduce reads grad, x and out and writes g (8), its elementwise pass reads g and x and writes dx (6); the
forked reduce reads grad2 too (2 more).  Prints one JSON line per shape, then the totals over the 15 forked sites.

Then, in a separate profiled run, one forward + backward of the rewritten ResNet-50 with and without the fork: kernels
per step and the number of torch add kernels (one per forked block output without the fork, none with it).

    python bench_bn_block.py [--iters N] [--batch B] [--no-profile]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

# (C, H = W, forked sites) of torchvision's ResNet-50: every block output but the last
SITES = [(256, 56, 3), (512, 28, 4), (1024, 14, 6), (2048, 7, 2)]


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


def sites(args, torch, eng):
    assert sum(s[2] for s in SITES) == 15
    tot = {"add_site_us": 0.0, "forked_us": 0.0}
    for c, hw, n_sites in SITES:
        g = torch.Generator(device="cuda").manual_seed(c + hw)
        shape = (args.batch, c, hw, hw)

        def cl(t):
            return t.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)

        x, out, g0, g1 = (cl(torch.randn(shape, device="cuda", generator=g)) for _ in range(4))
        out.relu_()
        w = torch.rand(c, device="cuda", generator=g).to(torch.bfloat16) + 0.5
        mean, invstd = torch.randn(c, device="cuda", generator=g), torch.rand(c, device="cuda", generator=g) + 0.5
        dx, dr = torch.empty_like(x), torch.empty_like(x)
        dw, db = torch.empty_like(w), torch.empty_like(w)

        def add_site():
            eng.bn_act_backward(g0 + g1, x, out, mean, invstd, w, None, dx, dw, db, dr)

        def forked():
            eng.bn_act_backward(g0, x, out, mean, invstd, w, None, dx, dw, db, dr, grad2=g1)

        t_add, t_fork = (_time(f, args.iters, torch) for f in (add_site, forked))
        n = x.numel()
        row = {"C": c, "HW": hw, "sites": n_sites, "add_site_us": round(t_add, 1), "forked_us": round(t_fork, 1),
               "add_site_TBps": round(20 * n / t_add / 1e6, 2), "forked_TBps": round(16 * n / t_fork / 1e6, 2),
               "GB_saved": round(4 * n / 1e9, 3)}
        print(json.dumps(row))
        tot["add_site_us"] += n_sites * t_add
        tot["forked_us"] += n_sites * t_fork
        del x, out, g0, g1, dx, dr
    return {k: round(v, 1) for k, v in tot.items()} | {"saved_us_per_step": round(tot["add_site_us"] - tot["forked_us"], 1)}


DOWNSAMPLE = [(256, 56), (512, 28), (1024, 14), (2048, 7)]


def downsample(args, torch, eng):
    """the forward of ResNet-50's 4 downsample sites: torch's BatchNorm on b, then the residual site reading its output
    (8 B/elem of b's statistics, apply and re-read beyond the site), against the two-BatchNorm site (4 B/elem: b's
    statistics read and its read in the apply)"""
    tot = {"torch_bn_site_us": 0.0, "two_bn_us": 0.0}
    for c, hw in DOWNSAMPLE:
        g = torch.Generator(device="cuda").manual_seed(c + hw)
        shape = (args.batch, c, hw, hw)
        x, r = (torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
                for _ in range(2))
        bn = torch.nn.BatchNorm2d(c).to(device="cuda", dtype=torch.bfloat16).to(memory_format=torch.channels_last)
        w, b = bn.weight.detach(), bn.bias.detach()
        rm, rv = torch.zeros(c, device="cuda"), torch.ones(c, device="cuda")
        rm2, rv2 = rm.clone(), rv.clone()
        out, mean, inv, mean2, inv2 = (torch.empty_like(x), *(torch.empty(c, device="cuda") for _ in range(4)))

        def unfused():
            with torch.no_grad():
                ident = bn(r)
            eng.bn_stats_act(x, ident, w, b, rm, rv, 0.1, 1e-5, out, mean, inv)

        def two_bn():
            eng.bn_stats_act(x, r, w, b, rm, rv, 0.1, 1e-5, out, mean, inv,
                             residual_bn=(w, b, rm2, rv2, 0.1, 1e-5, mean2, inv2))

        t_unf, t_two = (_time(f, args.iters, torch) for f in (unfused, two_bn))
        n = x.numel()
        print(json.dumps({"C": c, "HW": hw, "torch_bn_site_us": round(t_unf, 1), "two_bn_us": round(t_two, 1),
                          "two_bn_TBps": round(10 * n / t_two / 1e6, 2), "GB_saved": round(4 * n / 1e9, 3)}))
        tot["torch_bn_site_us"] += t_unf
        tot["two_bn_us"] += t_two
    return {k: round(v, 1) for k, v in tot.items()} | {"saved_us_per_step": round(tot["torch_bn_site_us"] - tot["two_bn_us"], 1)}


def profile(args, torch, eng):
    """kernels in one forward + backward of the rewritten ResNet-50, with and without the block-output fork"""
    from stoke_b200 import fuse, synthetic

    result = {}
    for fork in (False, True):
        torch.manual_seed(0)
        model = synthetic.resnet50().to(device="cuda", dtype=torch.bfloat16, memory_format=torch.channels_last)
        gm, n_required = fuse._trace(model)
        n_sites = fuse._rewrite(gm, eng)
        n_forks = fuse._fork(gm) if fork else 0
        gm.recompile()
        fwd = fuse.FusedForward(model, gm, n_required, n_sites)
        x = torch.randn(args.batch, 3, 224, 224, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        y = torch.randint(0, 1000, (args.batch,), device="cuda")
        lossf = torch.nn.CrossEntropyLoss()

        def step():
            lossf(fwd(x).float(), y).backward()

        for _ in range(2):
            step()
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            step()
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                 and "memset" not in e.name.lower() and "memcpy" not in e.name.lower()]
        adds = [n for n in names if "CUDAFunctor_add" in n or "AddFunctor" in n]
        result["fork" if fork else "no_fork"] = {"forked_sites": n_forks, "kernels": len(names), "add_kernels": len(adds)}
        del model, fwd, gm
        torch.cuda.empty_cache()
    return result


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--no-profile", action="store_true")
    args = ap.parse_args()
    import torch

    from stoke_b200.engine import get_engine

    if not torch.cuda.is_available():
        raise SystemExit("bench_bn_block.py needs a CUDA device")
    torch.cuda.set_device(0)
    eng = get_engine(0)
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": gpu, "batch": args.batch, "downsample_sites": 4, **downsample(args, torch, eng)}))
    print(json.dumps({"gpu": gpu, "batch": args.batch, "forked_sites": 15, **sites(args, torch, eng)}))
    if not args.no_profile:
        print(json.dumps({"gpu": gpu, "batch": args.batch, "forward_backward": profile(args, torch, eng)}))


if __name__ == "__main__":
    main()
