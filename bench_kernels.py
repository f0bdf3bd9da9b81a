# -*- coding: utf-8 -*-
"""Kernel-level roofline of the engine on one H100, on flat buffers of ResNet-50 size (25.6 M elements) and BERT-base size
(109.5 M elements):

  local route (the world-1 training path)   k_grad_norm (2 B/elem: one read of the raw bf16 bucket) and k_optim_step reading
                                            and zeroing the raw bucket (30 B/elem), timed separately and back to back
  main route                                k_grad_reduce at W=1 (6 B/elem algorithmic: read grad, write fp32 main grad; + 2
                                            for the bucket zeroing) and k_optim_step on fp32 main grads (30 B/elem)
  k_grad_accumulate                         the local no-sync micro-step

    python bench_kernels.py [--out kernels.json]

Timing: CUDA events on the launch stream around `iters` back-to-back launches after warm-up; every launch streams buffers
larger than the 50 MB L2 (BERT) or is preceded by an L2 flush write (ResNet-50, flagged in the output); achieved =
algorithmic bytes / time, peak = MEASURED_PEAKS.json hbm_gbs when present, else the H100 SXM data sheet (3.35 TB/s).
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--iters", type=int, default=30)
    args = ap.parse_args()
    from stoke_b200 import _lib
    from stoke_b200.engine import ClipSpec, get_engine
    from stoke_b200.optim import B200FusedOptimizer

    torch.cuda.set_device(0)
    eng = get_engine(0)
    peak = 3350.0   # H100 SXM data sheet, HBM3
    try:
        peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
    except OSError:
        pass
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    rows = []

    def timed(fn, nbytes, name, size_name, flush_l2):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        ms = []
        for _ in range(args.iters):
            if flush_l2:
                flush.fill_(1)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        ms.sort()
        med = ms[len(ms) // 2]
        row = {"kernel": name, "size": size_name, "us_median": med * 1e3, "us_min": ms[0] * 1e3, "bytes": nbytes,
               "achieved_gbs": nbytes / (med * 1e-3) / 1e9, "frac_of_measured_hbm_peak": nbytes / (med * 1e-3) / 1e9 / peak,
               "l2_flush_between_launches": bool(flush_l2)}
        rows.append(row)
        print(json.dumps(row), flush=True)

    class Flat(torch.nn.Module):
        def __init__(self, n):
            super().__init__()
            self.w = torch.nn.Parameter(torch.zeros(n))

    for size_name, n in (("resnet50_25.6M", 25_557_032), ("bert_base_109.5M", 109_483_778)):
        for optim_cls, kw, lp, tag in ((torch.optim.Adam, {"lr": 1e-3}, torch.bfloat16, "adam_bf16"),
                                       (torch.optim.Adam, {"lr": 1e-3}, None, "adam_fp32"),
                                       (torch.optim.SGD, {"lr": 0.1, "momentum": 0.9}, torch.bfloat16, "sgdm_bf16")):
            gsz = 2 if lp is not None else 4
            flush_l2 = n < 60_000_000
            per = {"adam_bf16": 30, "adam_fp32": 28, "sgdm_bf16": 22}[tag]
            for route in ("local", "main"):
                net = Flat(n).cuda()
                opt = B200FusedOptimizer(net, optim_cls, kw, engine=eng, grad_accum=2, route=route,
                                         clip=ClipSpec(_lib.CLIP_NORM, max_norm=1.0, norm_type=2.0), lp_dtype=lp)
                path = opt.path
                npad = path.n
                hyper = opt._hyper_of(opt.param_groups[0])

                def fill():
                    path.g_flat.copy_((torch.randn(path.n, device="cuda") * 1e-3).to(path.g_flat.dtype))

                fill()
                if route == "local":
                    # the norm pass reads the bucket and writes nothing: it can be timed in isolation
                    timed(lambda: path.after_backward(sync=True, unscale=False), npad * gsz, f"k_grad_norm[{tag}]",
                          size_name, flush_l2)
                    # the fused step consumes (zeroes) the bucket; its traffic does not depend on the values
                    timed(lambda: path.optimizer_step(hyper), npad * (per + (gsz - 4) + gsz), f"k_optim_step[raw,{tag}] (+epilogue)",
                          size_name, flush_l2)

                    def both():
                        path.after_backward(sync=True, unscale=False)
                        path.optimizer_step(hyper)

                    # back to back WITHOUT a flush in between: the step's read of the bucket can hit L2
                    timed(both, npad * (gsz + per + (gsz - 4) + gsz), f"k_grad_norm+k_optim_step[raw,{tag}]", size_name, flush_l2)
                else:
                    timed(lambda: path.after_backward(sync=True, unscale=False), npad * (gsz + 4), f"k_grad_reduce[W=1,{tag}]",
                          size_name, flush_l2)
                    fill()
                    timed(lambda: eng.grad_accumulate(path.G.ptr, path.model_dtype, path.ACC.ptr, npad, first=False, zero_grad=True),
                          npad * (gsz + 4 + 4 + gsz), f"k_grad_accumulate[{tag}]", size_name, flush_l2)
                    path.main_flat.copy_(torch.randn(path.n, device="cuda") * 1e-3)
                    timed(lambda: path.optimizer_step(hyper), npad * per, f"k_optim_step[main,{tag}] (+epilogue)", size_name, flush_l2)
                opt.close()
                del opt, path, net
                torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"peak_hbm_gbs": peak, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
