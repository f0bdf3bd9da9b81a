"""The block-output fork of the fuse_bn_act rewrite (stoke_b200/fuse.py) on the CPU: which residual sites return their
output once per user, and that the rewritten model (which takes the unfused fallback on the CPU, returning the same
tensor twice) computes exactly what the original does."""
import copy
import operator

import torch
import torchvision

from stoke_b200.fuse import BnAct, fuse_bn_act


def _forks(fwd):
    gm = fwd.graph_module
    forked = [n for n in gm.graph.nodes
              if n.op == "call_module" and isinstance(gm.get_submodule(n.target), BnAct) and gm.get_submodule(n.target).fork]
    for n in forked:   # each user reads its own output
        assert sorted(u.args[1] for u in n.users if u.target is operator.getitem) == [0, 1]
        assert all(len(u.users) == 1 for u in n.users)
    return len(forked)


def test_downsample_batchnorm_joins_the_residual_site():
    for name, two_bn in (("resnet50", 4), ("resnet18", 3)):
        model = getattr(torchvision.models, name)()
        fwd = fuse_bn_act(model, None)
        gm = fwd.graph_module
        acts = [gm.get_submodule(n.target) for n in gm.graph.nodes
                if n.op == "call_module" and isinstance(gm.get_submodule(n.target), BnAct)]
        rbns = [m.residual_bn for m in acts if m.residual_bn is not None]
        assert len(rbns) == two_bn, name
        # the user's downsample BatchNorms, shared, and no longer called on their own
        assert all(any(rb is blk.downsample[1] for rb in rbns) for layer in (model.layer1, model.layer2, model.layer3,
                                                                           model.layer4)
                   for blk in layer if blk.downsample is not None)
        assert not [n for n in gm.graph.nodes if n.op == "call_module" and n.target.endswith("downsample.1")]


def test_resnet_block_outputs_fork():
    # every block output but the last feeds the next block's conv1 and its identity or downsample conv
    assert _forks(fuse_bn_act(torchvision.models.resnet50(), None)) == 15
    assert _forks(fuse_bn_act(torchvision.models.resnet18(), None)) == 7


class Blocks(torch.nn.Module):
    """Two basic blocks; the first one's output has two users chosen by ``second``."""

    def __init__(self, second):
        super().__init__()
        self.second = second
        self.conv1 = torch.nn.Conv2d(8, 8, 3, padding=1)
        self.bn1 = torch.nn.BatchNorm2d(8)
        self.conv2 = torch.nn.Conv2d(8, 8, 3, padding=1)
        self.bn2 = torch.nn.BatchNorm2d(8)
        self.relu = torch.nn.ReLU(inplace=True)
        self.down = torch.nn.Conv2d(8, 8, 1)

    def forward(self, x):
        y = self.relu(self.bn1(self.conv1(x)) + x)          # the site that may fork
        z = self.bn2(self.conv2(y))
        if self.second == "identity":
            return self.relu(z + y)
        if self.second == "downsample":
            return self.relu(z + self.down(y))
        if self.second == "inplace":                         # y += ... mutates y: no fork
            y += z
            return y.detach()
        return self.relu(z + y), y.sum()                     # three users: no fork


def test_fork_only_for_two_reading_users():
    expect = {"identity": 1, "downsample": 1, "inplace": 0, "three": 0}
    for second, forks in expect.items():
        torch.manual_seed(0)
        ref = Blocks(second)
        mine = copy.deepcopy(ref)
        fwd = fuse_bn_act(mine, None)
        assert _forks(fwd) == forks, second
        x = torch.randn(2, 8, 6, 6).contiguous(memory_format=torch.channels_last)
        xa, xb = x.clone().requires_grad_(), x.clone().requires_grad_()
        a, b = ref(xa), fwd(xb)
        a, b = (a,) if torch.is_tensor(a) else a, (b,) if torch.is_tensor(b) else b
        assert all(torch.equal(u, v) for u, v in zip(a, b)), second
        if second == "inplace":   # the mutated ReLU output leaves nothing to differentiate
            continue
        sum(t.float().square().sum() for t in a).backward()
        sum(t.float().square().sum() for t in b).backward()
        assert torch.equal(xa.grad, xb.grad), second
        for (name, p), q in zip(ref.named_parameters(), mine.parameters()):
            assert (p.grad is None and q.grad is None) or torch.equal(p.grad, q.grad), (second, name)
        for (name, u), v in zip(ref.named_buffers(), mine.buffers()):
            assert torch.equal(u, v), (second, name)


def test_fallback_returns_one_tensor_twice():
    m = BnAct(torch.nn.BatchNorm2d(8), None, fork=True)
    x, r = torch.randn(2, 8, 3, 3), torch.randn(2, 8, 3, 3)
    a, b = m(x, r)
    assert a is b
