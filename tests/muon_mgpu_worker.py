"""Worker for the W = 2 test of tests/test_gpu_muon.py, launched through torch.distributed.run with one process per GPU:
``muon_mgpu_worker.py <out.json>``.  Every rank runs MuonWithAuxAdamW on the fused step with fairscale_oss asked for
(the state is replicated on the all-reduce route) on its own seeded bf16 gradients.  Rank 0 writes the route and whether
the two replicas' masters, momentum buffers, AdamW moments and bf16 copies are bit-identical."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main(out_path):
    from test_gpu_muon import SHAPES, Mats, _aux_kw

    from stoke_b200 import MuonWithAuxAdamW, synthetic
    from stoke_b200.engine import get_engine
    from stoke_b200.optim import B200FusedOptimizer

    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    torch.distributed.init_process_group("nccl", device_id=torch.device("cuda", local))
    eng = get_engine(local, rank, world)
    net = Mats(SHAPES).cuda()
    opt = B200FusedOptimizer(net, MuonWithAuxAdamW, _aux_kw(net), engine=eng, sharded=True, lp_dtype=torch.bfloat16)
    path = opt.path
    for step in range(4):
        for i, gv in enumerate(path.grad_views):
            g = synthetic.injected_grad(gv.numel(), rank, step * 100 + i, dtype=torch.bfloat16, scale=1e-2)
            gv.copy_(g.view(gv.shape).cuda())
        path.after_backward(sync=True, unscale=False)
        opt.step()
    eng.comm_check()
    mine = torch.cat([t.reshape(-1).view(torch.uint8) for t in
                      (path.gather_master(), path.m_flat, path.v_flat, path.p_flat, path.mu_x)])
    others = [torch.empty_like(mine) for _ in range(world)]
    torch.distributed.all_gather(others, mine)
    result = {"route": path.route, "replicas_identical": all(torch.equal(others[0], o) for o in others)}
    torch.distributed.barrier()
    if rank == 0:
        with open(out_path, "w") as f:
            json.dump(result, f)
    opt.close()
    torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main(sys.argv[1])
