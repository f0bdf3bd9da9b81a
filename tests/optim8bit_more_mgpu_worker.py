"""Worker for the W = 2 test of tests/test_gpu_optim8bit_more.py, launched through torch.distributed.run with one process
per GPU: ``optim8bit_more_mgpu_worker.py <Lion8bit | AdEMAMix8bit> <out.json>``.  Every rank runs the class on the fused
step with fairscale_oss asked for (the 8-bit state is replicated on the all-reduce route) on its own seeded bf16
gradients, and the class on CUDA fp32 copies of the initial master stepping on the mean gradient (what the world-1 step
sees).  Rank 0 writes the route, whether the two replicas' masters, codes, absmax and fp32 state are bit-identical, and
whether they equal the class's."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main(name, out_path):
    from test_gpu_optim8bit import SHAPES, Shapes
    from test_gpu_optim8bit_more import GROUPS, KW, _cls, _kwargs

    from stoke_b200 import synthetic
    from stoke_b200.engine import get_engine
    from stoke_b200.optim import B200FusedOptimizer

    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    torch.distributed.init_process_group("nccl", device_id=torch.device("cuda", local))
    eng = get_engine(local, rank, world)
    net = Shapes(SHAPES).cuda()
    opt = B200FusedOptimizer(net, _cls(name), _kwargs(net, GROUPS[name]), engine=eng, sharded=True,
                             lp_dtype=torch.bfloat16)
    path = opt.path
    ref = [torch.nn.Parameter(torch.empty_like(v).copy_(v)) for v in path.unflatten(path.gather_master())]
    ropt = _cls(name)([dict(KW, **extra, params=[ref[i] for i in idx]) for idx, extra in GROUPS[name]])
    for step in range(5):
        mean = []
        for i, gv in enumerate(path.grad_views):
            gs = [synthetic.injected_grad(gv.numel(), r, step * 100 + i, dtype=torch.bfloat16, scale=1e-2).view(gv.shape)
                  for r in range(world)]
            gv.copy_(gs[rank].cuda())
            mean.append((gs[0].float() + gs[1].float()).cuda() * 0.5)
        path.after_backward(sync=True, unscale=False)
        opt.step()
        for p, g in zip(ref, mean):
            p.grad = g
        ropt.step()
    eng.comm_check()
    views = path.q8_state_views()
    mine = torch.cat([path.gather_master().view(torch.uint8)] +
                     [v.contiguous().reshape(-1).view(torch.uint8) for d in views for v in d.values()])
    others = [torch.empty_like(mine) for _ in range(world)]
    torch.distributed.all_gather(others, mine)
    same_w1 = all(torch.equal(a.view(torch.int32), b.detach().view(torch.int32))
                  for a, b in zip(path.unflatten(path.gather_master()), ref))
    for d, p in zip(views, ref):
        same_w1 &= all(torch.equal(v, ropt.state[p][k]) for k, v in d.items())
    result = {"route": path.route, "replicas_identical": all(torch.equal(others[0], o) for o in others),
              "matches_world1": bool(same_w1)}
    torch.distributed.barrier()
    if rank == 0:
        with open(out_path, "w") as f:
            json.dump(result, f)
    opt.close()
    torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
