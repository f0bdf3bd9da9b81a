"""The BatchNorm2d -> [add] -> ReLU rewrite of stoke_b200/fuse.py on the CPU: which chains it fuses, that it shares the
user's modules, and that the rewritten model (which takes the unfused fallback on the CPU) computes exactly what the
original does -- outputs, gradients, running statistics and num_batches_tracked."""
import copy

import pytest
import torch
import torch.nn.functional as F
import torchvision

from stoke_b200.fuse import BnAct, fuse_bn_act


def _sites(fwd):
    gm = fwd.graph_module
    acts = [n for n in gm.graph.nodes if n.op == "call_module" and isinstance(gm.get_submodule(n.target), BnAct)]
    return len([n for n in acts if len(n.args) == 1]), len([n for n in acts if len(n.args) == 2])


def test_resnet50_sites():
    model = torchvision.models.resnet50()
    fwd = fuse_bn_act(model, None)
    gm = fwd.graph_module
    # stem + bn1 / bn2 of 16 bottlenecks feed a ReLU; bn3 feeds `out += identity` -> ReLU (the downsample BN is the residual)
    assert _sites(fwd) == (33, 16)
    assert fwd.fused_sites == 49
    assert not [n for n in gm.graph.nodes if n.op == "call_module" and isinstance(gm.get_submodule(n.target), torch.nn.ReLU)]


def test_resnet18_sites():
    assert _sites(fuse_bn_act(torchvision.models.resnet18(), None)) == (9, 8)


def test_shares_modules_and_keeps_state_dict():
    model = torchvision.models.resnet18()
    keys = list(model.state_dict().keys())
    gm = fuse_bn_act(model, None).graph_module
    assert list(model.state_dict().keys()) == keys
    assert gm.get_submodule("layer1.0.conv1") is model.layer1[0].conv1
    assert gm.layer1_0_bn1_act.bn is model.layer1[0].bn1
    assert gm.conv1.weight is model.conv1.weight


class TwoUsers(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = torch.nn.Conv2d(8, 8, 3, padding=1)
        self.bn = torch.nn.BatchNorm2d(8)
        self.bn2 = torch.nn.BatchNorm2d(8)

    def forward(self, x):
        y = self.bn(self.conv(x))
        z = torch.relu(self.bn2(x) + y)   # the add has one user, but its BN operand bn feeds the add and the return
        return torch.relu(y), z


def test_bn_with_two_users_is_left_alone():
    fwd = fuse_bn_act(TwoUsers(), None)
    gm = fwd.graph_module
    # bn has two users (relu and the add): never fused; bn2 -> add -> relu is, with bn's output as the residual
    assert _sites(fwd) == (0, 1)
    assert gm.graph.find_nodes(op="call_module", target="bn")


def test_nothing_to_fuse_or_untraceable():
    assert fuse_bn_act(torch.nn.Sequential(torch.nn.Linear(4, 4), torch.nn.ReLU()), None) is None

    class Branchy(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.bn = torch.nn.BatchNorm2d(8)

        def forward(self, x):
            return torch.relu(self.bn(x)) if x.sum() > 0 else x   # data-dependent control flow: fx cannot trace it

    assert fuse_bn_act(Branchy(), None) is None


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("momentum", [0.1, None])
def test_fallback_is_the_unfused_model(dtype, momentum):
    torch.manual_seed(0)
    ref = torchvision.models.resnet18(num_classes=10)
    for m in ref.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.momentum = momentum
            torch.nn.init.uniform_(m.weight, 0.5, 1.5)
            torch.nn.init.uniform_(m.bias, -0.5, 0.5)
    ref = ref.to(dtype=dtype, memory_format=torch.channels_last)
    mine = copy.deepcopy(ref)
    fwd = fuse_bn_act(mine, None)
    g = torch.Generator().manual_seed(1)
    for step in range(3):
        x = torch.randn(2, 3, 32, 32, generator=g).to(dtype).contiguous(memory_format=torch.channels_last)
        if step == 2:
            ref.eval(), mine.eval()
        a, b = ref(x), fwd(x)
        assert torch.equal(a, b)
        a.float().square().sum().backward()
        b.float().square().sum().backward()
        for (name, p), q in zip(ref.named_parameters(), mine.parameters()):
            assert torch.equal(p.grad, q.grad), name
        for (name, u), v in zip(ref.named_buffers(), mine.buffers()):
            assert torch.equal(u, v), name


class DropoutHead(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = torch.nn.Conv2d(3, 8, 3, padding=1)
        self.bn = torch.nn.BatchNorm2d(8)

    def forward(self, x, scale=None):
        x = F.relu(self.bn(self.conv(x)))
        if scale is not None:   # an optional argument: the graph is traced with it at its default
            x = x * scale
        return F.dropout(x, 0.5, training=self.training)   # a Python value read at trace time


def _pair(model_cls):
    torch.manual_seed(0)
    ref = model_cls()
    mine = copy.deepcopy(ref)
    return ref, mine, fuse_bn_act(mine, None)


def _same_call(ref, mine, fwd, *args, **kwargs):
    torch.manual_seed(5)
    a = ref(*args, **kwargs)
    torch.manual_seed(5)
    b = fwd(*args, **kwargs)
    assert torch.equal(a, b)
    return b


def test_graph_only_in_training_with_required_arguments():
    ref, mine, fwd = _pair(DropoutHead)
    assert _sites(fwd) == (1, 0)
    x = torch.randn(2, 3, 8, 8)
    _same_call(ref, mine, fwd, x)
    _same_call(ref, mine, fwd, x, 2.0)           # optional argument given: the module itself runs
    _same_call(ref, mine, fwd, x, scale=3.0)
    ref.eval(), mine.eval()
    _same_call(ref, mine, fwd, x)                # eval: the module itself runs, so no dropout is applied
    ref.train(), mine.train()
    ref.bn.eval(), mine.bn.eval()                # one submodule in eval is not what the graph was traced for
    _same_call(ref, mine, fwd, x)
    assert mine.training and not mine.bn.training   # tracing left the training flags as it found them


def test_hooks_still_fire():
    ref, mine, fwd = _pair(DropoutHead)
    seen = []
    mine.register_forward_hook(lambda m, i, o: seen.append("top"))
    mine.bn.register_forward_hook(lambda m, i, o: seen.append("bn"))
    _same_call(ref, mine, fwd, torch.randn(2, 3, 8, 8))
    assert seen == ["bn", "top"]


class SameOperand(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.bn = torch.nn.BatchNorm2d(8)

    def forward(self, x):
        y = self.bn(x)
        return torch.relu(y + y)


class InplaceAdds(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.bn = torch.nn.BatchNorm2d(8).to(torch.bfloat16)
        self.bn2 = torch.nn.BatchNorm2d(8).to(torch.bfloat16)

    def forward(self, x, r):
        out = self.bn(x)
        out += r                     # bf16 += fp32 stays bf16
        out = torch.relu(out)
        identity = r
        identity += self.bn2(out)    # mutates r (BatchNorm on the right of +=): never fused
        return torch.relu(identity), r


def test_add_sites_that_are_skipped_or_keep_inplace_semantics():
    assert fuse_bn_act(SameOperand(), None) is None   # relu(y + y): both operands are the BatchNorm, nothing to fuse
    ref, mine, fwd = _pair(InplaceAdds)
    assert _sites(fwd) == (0, 1)
    x = torch.randn(2, 8, 4, 4).to(torch.bfloat16)
    r1 = torch.randn(2, 8, 4, 4)
    r2 = r1.clone()
    a, b = ref(x, r1), fwd(x, r2)
    assert all(torch.equal(u, v) and u.dtype == v.dtype for u, v in zip(a, b))
    assert torch.equal(r1, r2)
