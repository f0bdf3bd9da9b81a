"""Worker for the W = 2 test of tests/test_gpu_rmsprop_tf.py, launched through torch.distributed.run with one process per
GPU.  Every rank runs RMSpropTF twice on identical seeded gradients -- sharded (fairscale_oss: ZeRO-1 with the in-kernel
parameter all-gather; square_avg, momentum_buffer and grad_avg split by the same segments) and replicated (all-reduce
route) -- with a centered momentum group and a plain group, and rank 0 writes whether the final weights and the gathered
state_dicts are bit-identical."""
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
    from stoke_b200.optim import B200FusedOptimizer, RMSpropTF

    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    torch.distributed.init_process_group("nccl", device_id=torch.device("cuda", local))
    eng = get_engine(local, rank, world)
    runs = {}
    for sharded, route in ((True, "sharded"), (False, "allreduce")):
        torch.manual_seed(1234)
        net = OddNet(scale=3).cuda()
        ps = list(net.parameters())
        kw = {"lr": 1e-2, "alpha": 0.9, "eps": 1e-3, "momentum": 0.9, "weight_decay": 1e-5,
              "params": [dict(params=ps[:3], centered=True),
                         dict(params=ps[3:], momentum=0.0, weight_decay=0.01, decoupled_decay=True)]}
        opt = B200FusedOptimizer(net, RMSpropTF, kw, engine=eng, sharded=sharded, lp_dtype=torch.bfloat16, route=route)
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
                        for j, st in sd["state"].items()})
        opt.close()
        del opt, path, net

    (r_s, w_s, p_s, st_s), (r_r, w_r, p_r, st_r) = runs["sharded"], runs["allreduce"]
    same_state = st_s.keys() == st_r.keys() and all(
        st_s[j].keys() == st_r[j].keys() and all(torch.equal(st_s[j][k], st_r[j][k]) for k in st_s[j]) for j in st_s)
    result = {"sharded_route": r_s, "replicated_route": r_r,
              "weights_identical": bool(torch.equal(w_s, w_r) and torch.equal(p_s, p_r)),
              "state_identical": bool(same_state)}
    torch.distributed.barrier()
    if rank == 0:
        with open(out_path, "w") as f:
            json.dump(result, f)
    torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main(sys.argv[1])
