"""The BatchNorm2d -> SiLU / Hardswish / ReLU6 sites of the fuse_bn_act rewrite (stoke_b200/fuse.py) on the CPU: how many
of each kind it finds in torchvision's EfficientNet and MobileNet models, that ResNet-50 keeps its ReLU sites, the
module, functional and in-place forms, and that rewritten EfficientNet-B0 and MobileNetV3-Small (which take the unfused
fallback on the CPU) compute exactly what the originals do over two training steps."""
import copy

import pytest
import torch
import torch.nn.functional as F
import torchvision

from stoke_b200._lib import ACT_HARDSWISH, ACT_RELU, ACT_RELU6, ACT_SILU
from stoke_b200.fuse import BnAct, fuse_bn_act


def _kinds(fwd):
    """{kind: number of BnAct sites}; ReLU sites split into (without, with) a residual"""
    gm = fwd.graph_module
    out = {}
    for n in gm.graph.nodes:
        if n.op == "call_module" and isinstance(gm.get_submodule(n.target), BnAct):
            kind = gm.get_submodule(n.target).act
            key = (kind, len(n.args) == 2) if kind == ACT_RELU else kind
            out[key] = out.get(key, 0) + 1
    return out


# single-user BatchNorm2d -> activation chains of the torchvision models in training mode
MODEL_SITES = {
    "efficientnet_b0": {ACT_SILU: 33},
    "efficientnet_v2_s": {ACT_SILU: 72},
    "mobilenet_v2": {ACT_RELU6: 35},
    "mobilenet_v3_large": {ACT_HARDSWISH: 20, (ACT_RELU, False): 11},
    "mobilenet_v3_small": {ACT_HARDSWISH: 18, (ACT_RELU, False): 5},
    "resnet50": {(ACT_RELU, False): 33, (ACT_RELU, True): 16},
}


@pytest.mark.parametrize("name", sorted(MODEL_SITES))
def test_model_sites(name):
    fwd = fuse_bn_act(getattr(torchvision.models, name)(), None)
    assert _kinds(fwd) == MODEL_SITES[name]
    assert fwd.fused_sites == sum(MODEL_SITES[name].values())
    gm = fwd.graph_module
    left = [n for n in gm.graph.nodes if n.op == "call_module"
            and type(gm.get_submodule(n.target)) in (torch.nn.SiLU, torch.nn.Hardswish, torch.nn.ReLU6)]
    assert not [n for n in left if n.args[0].op == "call_module"
                and type(gm.get_submodule(n.args[0].target)) is torch.nn.BatchNorm2d]


class Forms(torch.nn.Module):
    """every form of every activation after its own BatchNorm, and one BatchNorm -> SiLU -> add the rewrite must not take
    for a residual site"""

    FORMS = [
        (ACT_SILU, lambda: torch.nn.SiLU()), (ACT_SILU, lambda: torch.nn.SiLU(inplace=True)),
        (ACT_SILU, lambda: F.silu), (ACT_SILU, lambda: lambda y: F.silu(y, inplace=True)),
        (ACT_SILU, lambda: lambda y: F.silu(y, True)),
        (ACT_HARDSWISH, lambda: torch.nn.Hardswish()), (ACT_HARDSWISH, lambda: torch.nn.Hardswish(inplace=True)),
        (ACT_HARDSWISH, lambda: F.hardswish), (ACT_HARDSWISH, lambda: lambda y: F.hardswish(y, inplace=True)),
        (ACT_RELU6, lambda: torch.nn.ReLU6()), (ACT_RELU6, lambda: torch.nn.ReLU6(inplace=True)),
        (ACT_RELU6, lambda: F.relu6), (ACT_RELU6, lambda: lambda y: F.relu6(y, inplace=True)),
    ]

    def __init__(self):
        super().__init__()
        self.bns = torch.nn.ModuleList(torch.nn.BatchNorm2d(8) for _ in range(len(self.FORMS)))
        self.acts = [make() for _, make in self.FORMS]
        self.mods = torch.nn.ModuleList(a for a in self.acts if isinstance(a, torch.nn.Module))
        self.bn_res = torch.nn.BatchNorm2d(8)

    def forward(self, x):
        outs = []
        for bn, act in zip(self.bns, self.acts):
            outs.append(act(bn(x)))
        outs.append(F.silu(self.bn_res(x) + x))   # the BatchNorm's user is the add: left alone
        return torch.stack(outs).sum(0)


def test_module_functional_and_inplace_forms():
    torch.manual_seed(0)
    ref = Forms()
    mine = copy.deepcopy(ref)
    fwd = fuse_bn_act(mine, None)
    kinds = [k for k, _ in Forms.FORMS]
    assert _kinds(fwd) == {k: kinds.count(k) for k in set(kinds)}
    gm = fwd.graph_module
    assert gm.graph.find_nodes(op="call_module", target="bn_res")
    x = torch.randn(4, 8, 5, 5) * 4
    a, b = ref(x), fwd(x)
    assert torch.equal(a, b)
    a.square().sum().backward()
    b.square().sum().backward()
    for (name, p), q in zip(ref.named_parameters(), mine.parameters()):
        assert torch.equal(p.grad, q.grad), name


class TwoUsersSiLU(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.bn = torch.nn.BatchNorm2d(8)
        self.act = torch.nn.SiLU()

    def forward(self, x):
        y = self.bn(x)
        return self.act(y), y


def test_bn_with_two_users_is_left_alone():
    assert fuse_bn_act(TwoUsersSiLU(), None) is None


class HardtanhNotRelu6(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.bn = torch.nn.BatchNorm2d(8)
        self.act = torch.nn.Hardtanh(0.0, 6.0)   # the same function, but not one of the matched forms

    def forward(self, x):
        return self.act(self.bn(x))


def test_only_the_listed_forms_are_matched():
    assert fuse_bn_act(HardtanhNotRelu6(), None) is None


def test_bnact_rejects_a_residual_for_other_activations():
    m = BnAct(torch.nn.BatchNorm2d(8), None, act=ACT_SILU)
    x = torch.randn(2, 8, 3, 3)
    with pytest.raises(ValueError):
        m(x, x)
    with pytest.raises(ValueError):
        BnAct(torch.nn.BatchNorm2d(8), None, act=7)


@pytest.mark.parametrize("name", ["efficientnet_b0", "mobilenet_v3_small"])
def test_rewritten_model_is_the_unfused_model(name):
    torch.manual_seed(0)
    ref = getattr(torchvision.models, name)(num_classes=10)
    for m in ref.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            torch.nn.init.uniform_(m.weight, 0.5, 1.5)
            torch.nn.init.uniform_(m.bias, -0.5, 0.5)
    ref = ref.to(memory_format=torch.channels_last)
    mine = copy.deepcopy(ref)
    fwd = fuse_bn_act(mine, None)
    assert fwd is not None
    g = torch.Generator().manual_seed(1)
    for _ in range(2):
        x = torch.randn(2, 3, 64, 64, generator=g).contiguous(memory_format=torch.channels_last)
        torch.manual_seed(7)   # dropout and stochastic depth draw the same masks in both models
        a = ref(x)
        torch.manual_seed(7)
        b = fwd(x)
        assert torch.equal(a, b)
        a.square().sum().backward()
        b.square().sum().backward()
        for (pname, p), q in zip(ref.named_parameters(), mine.parameters()):
            assert torch.equal(p.grad, q.grad), pname
        for (bname, u), v in zip(ref.named_buffers(), mine.buffers()):
            assert torch.equal(u, v), bname
    assert all(int(m.num_batches_tracked) == 2 for m in mine.modules() if isinstance(m, torch.nn.BatchNorm2d))


@pytest.mark.parametrize("fn", [F.silu, F.hardswish, F.relu6])
@pytest.mark.parametrize("inplace", [False, True])
def test_positional_inplace_argument(fn, inplace):
    """a graph that records ``f(y, inplace)`` positionally (fx's tracer records it by keyword) keeps ``inplace`` bound
    by name in BnAct's unfused fallback"""
    from stoke_b200.fuse import _rewrite

    root = torch.nn.Module()
    root.bn = torch.nn.BatchNorm2d(8)
    graph = torch.fx.Graph()
    x = graph.placeholder("x")
    graph.output(graph.call_function(fn, (graph.call_module("bn", (x,)), inplace)))
    gm = torch.fx.GraphModule(root, graph)
    ref = copy.deepcopy(root.bn)
    assert _rewrite(gm, None) == 1
    gm.recompile()
    inp = torch.randn(2, 8, 3, 3) * 4
    assert torch.equal(gm(inp), fn(ref(inp)))


def test_site_shapes_on_the_meta_device():
    from stoke_b200.fuse import site_shapes

    with torch.device("meta"):
        fwd = fuse_bn_act(torchvision.models.mobilenet_v3_small(), None)
        sites = site_shapes(fwd, torch.empty(2, 3, 224, 224))
    assert sum(sites.values()) == fwd.fused_sites == 23
    assert sites[(ACT_HARDSWISH, 16, 112, 112, 0.001, 0.01)] == 1
    assert {k[0] for k in sites} == {ACT_HARDSWISH, ACT_RELU}
