"""Worker for the W = 2 LAMB / LARS test of tests/test_gpu_layerwise.py, launched through torch.distributed.run with one
process per GPU.  Every rank steps each class with fairscale_oss asked for (the state stays replicated: the all-reduce
route) on seeded per-rank gradients; rank 0 writes, per class, whether the replicas' masters and state are bit-identical
and the relative L2 error of the masters against the W = 1 oracle fed the same per-rank gradients."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))


def run(kind, eng, rank, world):
    from engine_oracle import OracleEngine
    from test_gpu_engine import OddNet, _oracle_flat, _rel

    from stoke_b200 import synthetic
    from stoke_b200.optim import LAMB, LARS, B200FusedOptimizer

    cls, kw = (LAMB, {"lr": 1e-2, "weight_decay": 0.01}) if kind == "lamb" else (LARS, {"lr": 0.5, "weight_decay": 1e-4})
    torch.manual_seed(1234)
    net = OddNet(scale=3).cuda()
    init = [p.detach().cpu().clone() for p in net.parameters()]
    opt = B200FusedOptimizer(net, cls, kw, engine=eng, sharded=True, lp_dtype=torch.bfloat16)
    path = opt.path
    oracle = OracleEngine(init, world, cls, kw)
    for step in range(8):
        per_rank = []
        for r in range(world):
            per_rank.append([synthetic.injected_grad(gv.numel(), r, step * 100 + i, dtype=torch.bfloat16).float()
                             for i, gv in enumerate(path.grad_views)])
        for i, gv in enumerate(path.grad_views):
            gv.copy_(per_rank[rank][i].to(torch.bfloat16).view(gv.shape).cuda())
        oracle.micro_step(per_rank)
        path.after_backward(sync=True, unscale=False)
        opt.step()
        oracle.step()
    eng.comm_check()
    master = path.gather_master()
    state = path.m_flat.clone()
    gathered_m = [torch.empty_like(master) for _ in range(world)]
    gathered_s = [torch.empty_like(state) for _ in range(world)]
    torch.distributed.all_gather(gathered_m, master)
    torch.distributed.all_gather(gathered_s, state)
    same = all(torch.equal(gathered_m[0].view(torch.int32), m.view(torch.int32)) for m in gathered_m) and \
        all(torch.equal(gathered_s[0].view(torch.int32), s.view(torch.int32)) for s in gathered_s)
    rel = _rel(master.cpu(), _oracle_flat(path, oracle.weights()))
    res = {"route": path.route, "replicas_identical": bool(same), "rel_vs_oracle": rel}
    opt.close()
    torch.distributed.barrier()
    return res


def main(out_path):
    from stoke_b200.engine import get_engine

    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    torch.distributed.init_process_group("nccl", device_id=torch.device("cuda", local))
    eng = get_engine(local, rank, world)
    res = {kind: run(kind, eng, rank, world) for kind in ("lamb", "lars")}
    if rank == 0:
        with open(out_path, "w") as f:
            json.dump(res, f)
    torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main(sys.argv[1])
