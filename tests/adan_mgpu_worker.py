"""Worker for the W = 2 test of tests/test_gpu_adan.py, launched through torch.distributed.run with one process per GPU.
Every rank runs Adan twice on identical seeded gradients -- sharded (fairscale_oss: ZeRO-1 with the in-kernel parameter
all-gather; exp_avg, exp_avg_sq, exp_avg_diff and neg_pre_grad split by the same segments) and replicated (all-reduce
route) -- with a proximal group and a no_prox group, and rank 0 writes whether the final weights, the gathered
state_dicts and the groups' step counts are identical."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main(out_path):
    from test_gpu_engine import OddNet

    from stoke_b200 import synthetic
    from stoke_b200.engine import get_engine
    from stoke_b200.optim import Adan, B200FusedOptimizer

    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    torch.distributed.init_process_group("nccl", device_id=torch.device("cuda", local))
    eng = get_engine(local, rank, world)
    runs = {}
    for sharded, route in ((True, "sharded"), (False, "allreduce")):
        torch.manual_seed(1234)
        net = OddNet(scale=3).cuda()
        ps = list(net.parameters())
        kw = {"lr": 1e-2, "betas": (0.98, 0.92, 0.99), "weight_decay": 0.02,
              "params": [dict(params=ps[:3]), dict(params=ps[3:], no_prox=True, betas=(0.9, 0.9, 0.999))]}
        opt = B200FusedOptimizer(net, Adan, kw, engine=eng, sharded=sharded, lp_dtype=torch.bfloat16, route=route)
        path = opt.path
        for step in range(7):
            for i, gv in enumerate(path.grad_views):
                gv.copy_(synthetic.injected_grad(gv.numel(), rank, step * 100 + i, dtype=torch.bfloat16).view(gv.shape).cuda())
            path.after_backward(sync=True, unscale=False)
            opt.step()
        eng.comm_check()
        sd = opt.state_dict()
        runs[route] = (path.route, path.gather_master().cpu(), path.p_flat.cpu().clone(),
                       {j: {k: (v.cpu().clone() if torch.is_tensor(v) else v) for k, v in st.items()}
                        for j, st in sd["state"].items()}, [g["step"] for g in sd["param_groups"]])
        opt.close()
        del opt, path, net

    (r_s, w_s, p_s, st_s, k_s), (r_r, w_r, p_r, st_r, k_r) = runs["sharded"], runs["allreduce"]
    same_state = st_s.keys() == st_r.keys() and all(
        st_s[j].keys() == st_r[j].keys() and all(torch.equal(st_s[j][k], st_r[j][k]) for k in st_s[j]) for j in st_s)
    result = {"sharded_route": r_s, "replicated_route": r_r,
              "weights_identical": bool(torch.equal(w_s, w_r) and torch.equal(p_s, p_r)),
              "state_identical": bool(same_state and k_s == k_r == [7, 7])}
    torch.distributed.barrier()
    if rank == 0:
        with open(out_path, "w") as f:
            json.dump(result, f)
    torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main(sys.argv[1])
