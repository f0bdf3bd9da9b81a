"""Worker for the W = 2 weight-average test of tests/test_gpu_weight_average.py, launched through torch.distributed.run
with one process per GPU.  On the sharded route (each rank averages its own shard of the master) and on the all-reduce
route (every rank averages all of it), Adam on a bf16 model with seeded per-rank gradients and an EMA every step.
Every rank checks, after every step, that the gathered average equals AveragedModel over the gathered master; that
``state_dict()`` (called on every rank) holds the same values under the model's names; that ``applied()`` puts the
average's bf16 cast into P and restores P bit for bit; and that loading a checkpoint taken mid-run brings back that
average and its count.  Rank 0 writes whether every rank saw every check pass."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _same(a, b):
    return a.dtype == b.dtype and torch.equal(a.contiguous().view(torch.int16 if a.element_size() == 2 else torch.int32),
                                              b.contiguous().view(torch.int16 if b.element_size() == 2 else torch.int32))


def run(route, eng, rank, world):
    from torch.optim.swa_utils import AveragedModel, get_ema_multi_avg_fn
    from test_gpu_engine import OddNet

    import stoke_b200 as sb
    from stoke_b200 import synthetic
    from stoke_b200.optim import B200FusedOptimizer
    from stoke_b200.weight_average import WeightAverage

    torch.manual_seed(1234)
    net = OddNet(scale=3).cuda()
    opt = B200FusedOptimizer(net, torch.optim.Adam, {"lr": 1e-2}, engine=eng, sharded=route == "sharded",
                             lp_dtype=torch.bfloat16, route=route)
    path = opt.path
    wa = WeightAverage(sb.WeightAverageConfig(decay=0.9), path, net)
    holder = torch.nn.ParameterList([torch.nn.Parameter(v.clone()) for v in path.unflatten(path.gather_master())])
    ref = AveragedModel(holder, multi_avg_fn=get_ema_multi_avg_fn(0.9))
    checks = {"avg_each_step": True, "state_dict": True, "applied": True, "restored": True, "load": True}
    ckpt = ckpt_avg = None
    for step in range(1, 7):
        for i, gv in enumerate(path.grad_views):
            g = synthetic.injected_grad(gv.numel(), rank, step * 100 + i, dtype=torch.bfloat16)
            gv.copy_(g.view(gv.shape).cuda())
        path.after_backward(sync=True, unscale=False)
        wa._schedule(step)
        opt.step()
        with torch.no_grad():
            for p, v in zip(holder, path.unflatten(path.gather_master())):
                p.copy_(v)
        ref.update_parameters(holder)
        got = path.unflatten(path.gather_avg())
        checks["avg_each_step"] &= all(_same(a, r.detach()) for a, r in zip(got, ref.module.parameters()))
        if step == 3:
            ckpt, ckpt_avg = wa._checkpoint(), path.gather_avg()
    eng.comm_check()

    sd = wa.state_dict()
    for p, r in zip(path.params, ref.module.parameters()):
        checks["state_dict"] &= _same(sd[wa._name_of[id(p)]], r.detach())

    before = path.p_flat.clone()
    cast = path.gather_avg().to(path.p_flat.dtype)
    with wa.applied():
        torch.cuda.synchronize()
        checks["applied"] &= _same(path.p_flat, cast)
    torch.cuda.synchronize()
    checks["restored"] &= _same(path.p_flat, before)

    wa._load_checkpoint(ckpt)
    checks["load"] &= wa.n_averaged == 3 and _same(path.gather_avg(), ckpt_avg)

    flags = torch.tensor([int(v) for v in checks.values()], dtype=torch.int32, device="cuda")
    torch.distributed.all_reduce(flags, op=torch.distributed.ReduceOp.MIN)
    res = dict(zip(checks, (bool(v) for v in flags.tolist())), route=path.route, n_local=path.n_local, n=path.n)
    opt.close()
    torch.distributed.barrier()
    return res


def main(out_path):
    from stoke_b200.engine import get_engine

    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    torch.distributed.init_process_group("nccl", device_id=torch.device("cuda", local))
    eng = get_engine(local, rank, world)
    res = {route: run(route, eng, rank, world) for route in ("sharded", "allreduce")}
    if rank == 0:
        with open(out_path, "w") as f:
            json.dump(res, f)
    torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main(sys.argv[1])
