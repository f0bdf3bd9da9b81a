"""torch.optim.Muon and MuonWithAuxAdamW (CPU): the class against the float64 transcription of tests/muon_ref.py and,
bit for bit, against torch.optim.Muon and torch.optim.AdamW; the conv reshape; argument validation; state layout,
routing (8 groups fused, 9 not; the classes that stay on the stock route stay there); the fused step's descriptor table,
C structs and FLOP count."""
import ctypes as C

import pytest
import torch

import muon_ref as mr
from stoke_b200 import MuonWithAuxAdamW, _lib, layout
from stoke_b200 import optim as O

needs_muon = pytest.mark.skipif(not hasattr(torch.optim, "Muon"), reason="torch.optim.Muon needs torch >= 2.9")


def _params(shapes, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.nn.Parameter(torch.randn(s, generator=g) * 0.1) for s in shapes]


def _grads(params, step, scale=1e-2):
    g = torch.Generator().manual_seed(100 + step)
    return [torch.randn(p.shape, generator=g) * scale for p in params]


MUON_SHAPES = [(8, 12), (20, 6), (1, 9), (9, 1), (33, 70)]


@needs_muon
@pytest.mark.parametrize("kw", [{}, {"nesterov": False, "weight_decay": 0.0, "momentum": 0.9},
                                {"adjust_lr_fn": "match_rms_adamw", "lr": 0.02, "ns_steps": 3},
                                {"adjust_lr_fn": "original", "ns_coefficients": (2.0, -1.5, 0.5), "eps": 1e-5}])
def test_muon_half_is_torch_muon_bit_for_bit(kw):
    """Muon groups of MuonWithAuxAdamW on 2-D parameters equal torch.optim.Muon bit for bit on CPU fp32 over 4 steps,
    with one parameter left without a gradient at step 2 (no state created, nothing touched)."""
    a, b = _params(MUON_SHAPES), _params(MUON_SHAPES)
    ta = torch.optim.Muon(a, **kw)
    tb = MuonWithAuxAdamW([dict(params=b, use_muon=True, **kw)])
    for step in range(4):
        for i, (p, q, g) in enumerate(zip(a, b, _grads(a, step))):
            skip = step < 2 and i == 2
            p.grad = None if skip else g.clone()
            q.grad = None if skip else g.clone()
        ta.step()
        tb.step()
        for p, q in zip(a, b):
            assert torch.equal(p, q)
            assert torch.equal(ta.state[p]["momentum_buffer"], tb.state[q]["momentum_buffer"]) if p in ta.state \
                else q not in tb.state
    assert list(tb.state_dict()["state"][0]) == ["momentum_buffer"]


def test_adamw_half_is_torch_adamw_bit_for_bit():
    """AdamW groups equal torch.optim.AdamW(foreach=False) bit for bit on CPU fp32, state keys and step included."""
    shapes = [(7,), (5, 3), (2, 3, 4)]
    kw = dict(lr=1e-2, betas=(0.8, 0.95), eps=1e-6, weight_decay=0.05)
    a, b = _params(shapes), _params(shapes)
    ta = torch.optim.AdamW(a, foreach=False, **kw)
    tb = MuonWithAuxAdamW([dict(params=b, use_muon=False, **kw)])
    for step in range(4):
        for p, q, g in zip(a, b, _grads(a, step)):
            p.grad, q.grad = g.clone(), g.clone()
        ta.step()
        tb.step()
    for p, q in zip(a, b):
        assert torch.equal(p, q)
        for k in ("step", "exp_avg", "exp_avg_sq"):
            assert torch.equal(ta.state[p][k], tb.state[q][k]), k
    assert list(tb.state_dict()["state"][0]) == ["step", "exp_avg", "exp_avg_sq"]


def test_class_against_the_float64_transcription():
    """One step of both halves against tests/muon_ref.py in float64: the momentum buffer and the AdamW state to fp32
    rounding; the Muon update to the bf16 Newton-Schulz error (2^-5 of its norm, per parameter)."""
    shapes = [(16, 24), (40, 12), (6, 3, 3, 3)]
    aux_shapes = [(24,), (12, 4)]
    mk = dict(lr=0.02, weight_decay=0.1, momentum=0.9, nesterov=True, ns_coefficients=mr.COEFFS, eps=1e-7, ns_steps=5,
              adjust_lr_fn="match_rms_adamw")
    ak = dict(lr=1e-2, betas=(0.9, 0.99), eps=1e-8, weight_decay=0.01)
    ps, qs = _params(shapes), _params(aux_shapes, 1)
    w0 = [p.detach().clone() for p in ps + qs]
    opt = MuonWithAuxAdamW([dict(params=ps, use_muon=True, **mk), dict(params=qs, use_muon=False, **ak)])
    bufs = [torch.zeros_like(p) for p in ps]
    for step in range(2):
        grads = _grads(ps + qs, step)
        for p, g in zip(ps + qs, grads):
            p.grad = g
        opt.step()
        for i, p in enumerate(ps):
            want, bufs[i] = mr.muon_step64(w0[i], bufs[i], grads[i], mk)
            assert torch.allclose(opt.state[p]["momentum_buffer"].double(), bufs[i], rtol=1e-6, atol=1e-9)
            upd = want - w0[i].double() * (1 - mk["lr"] * mk["weight_decay"])
            err = (p.detach().double() - want).norm() / upd.norm()
            assert err < 2 ** -5, (i, float(err))
            w0[i] = p.detach().clone()
        for j, q in enumerate(qs):
            st = opt.state[q]
            k = len(ps) + j
            m0 = st["exp_avg"].double() if step else torch.zeros_like(q, dtype=torch.float64)
            if step == 0:
                w, m, v = mr.adamw_step64(w0[k], m0, m0, grads[k], 1, ak)
            else:
                w, m, v = mr.adamw_step64(w0[k], prev[j][0], prev[j][1], grads[k], 2, ak)
            assert torch.allclose(q.detach().double(), w, rtol=1e-6, atol=1e-8)
            assert torch.allclose(st["exp_avg"].double(), m, rtol=1e-5, atol=1e-10)
            assert torch.allclose(st["exp_avg_sq"].double(), v, rtol=1e-5, atol=1e-14)
        prev = [(opt.state[q]["exp_avg"].double().clone(), opt.state[q]["exp_avg_sq"].double().clone()) for q in qs]
        w0[len(ps):] = [q.detach().clone() for q in qs]


def test_conv_weight_is_its_reshaped_matrix():
    """A (out, in, kh, kw) weight steps as the (out, in kh kw) matrix: equal bit for bit to torch.optim.Muon on that
    2-D matrix, for a contiguous and a channels-last weight, momentum buffer included (in the weight's shape)."""
    for fmt in (torch.contiguous_format, torch.channels_last):
        w = _params([(12, 4, 3, 3)], 3)[0]
        conv = torch.nn.Parameter(w.detach().clone().contiguous(memory_format=fmt))
        mat = torch.nn.Parameter(w.detach().clone().reshape(12, -1))
        a = MuonWithAuxAdamW([dict(params=[conv], use_muon=True, lr=0.05)])
        b = torch.optim.Muon([mat], lr=0.05) if hasattr(torch.optim, "Muon") else None
        for step in range(3):
            g = _grads([conv], step)[0]
            conv.grad = g.contiguous(memory_format=fmt)
            mat.grad = g.reshape(12, -1).clone()
            a.step()
            if b is not None:
                b.step()
        assert conv.is_contiguous(memory_format=fmt)
        assert a.state[conv]["momentum_buffer"].shape == (12, 4, 3, 3)
        if b is not None:
            assert torch.equal(conv.detach().reshape(12, -1), mat.detach())
            assert torch.equal(a.state[conv]["momentum_buffer"].reshape(12, -1), b.state[mat]["momentum_buffer"])


def test_argument_validation():
    p2, p1 = torch.nn.Parameter(torch.zeros(3, 4)), torch.nn.Parameter(torch.zeros(3))
    with pytest.raises(ValueError, match="use_muon"):
        MuonWithAuxAdamW([dict(params=[p2])])
    with pytest.raises(ValueError, match="2 or more dims"):
        MuonWithAuxAdamW([dict(params=[p1], use_muon=True)])
    for bad in (dict(lr=-1.0), dict(weight_decay=-0.1), dict(momentum=-0.5), dict(adjust_lr_fn="nope"),
                dict(ns_steps=100), dict(ns_coefficients=(1.0, 2.0)), dict(eps=-1.0)):
        with pytest.raises(ValueError):
            MuonWithAuxAdamW([dict(params=[p2], use_muon=True, **bad)])
    for bad in (dict(betas=(1.0, 0.9)), dict(betas=(0.9, -0.1)), dict(lr=-1.0), dict(eps=-1e-8)):
        with pytest.raises(ValueError):
            MuonWithAuxAdamW([dict(params=[p1], use_muon=False, **bad)])
    opt = MuonWithAuxAdamW([dict(params=[p2], use_muon=True), dict(params=[p1], use_muon=False)])
    g0, g1 = opt.param_groups
    assert (g0["lr"], g0["weight_decay"], g0["momentum"], g0["nesterov"], g0["ns_steps"], g0["eps"]) == \
        (1e-3, 0.1, 0.95, True, 5, 1e-7) and g0["adjust_lr_fn"] is None
    assert (g1["lr"], g1["betas"], g1["eps"], g1["weight_decay"]) == (1e-3, (0.9, 0.999), 1e-8, 1e-2)


@needs_muon
def test_lr_ratio_is_torchs():
    from torch.optim._muon import _adjust_lr

    for fn in (None, "original", "match_rms_adamw"):
        for r, c in [(3, 7), (7, 3), (768, 3072), (3072, 768), (1, 9), (64, 576)]:
            assert O.muon_lr_ratio(fn, r, c) == _adjust_lr(1.0, fn, torch.Size((r, c))) == mr.lr_ratio(fn, r, c)


def test_state_layout_buffers_and_hypers():
    lay = O._STATE_LAYOUT[O._MUON]
    muon_g, aux_g = {"use_muon": True}, {"use_muon": False}
    assert O.state_buffers(lay, [muon_g]) == {"M": 0.0, "V": None, "M2": None}
    assert O.state_buffers(lay, [{}]) == {"M": 0.0, "V": None, "M2": None}    # torch.optim.Muon's groups
    assert O.state_buffers(lay, [muon_g, aux_g]) == {"M": 0.0, "V": 0.0, "M2": None}
    assert lay.unstepped == "omit"
    g = dict(O._MUON_DEFAULTS, use_muon=True)
    m, h = O._muon_hyper(g)
    assert (m.lr, m.weight_decay, m.momentum, m.eps, m.nesterov, m.ns_steps) == (1e-3, 0.1, 0.95, 1e-7, 1, 5)
    assert (m.ns_a, m.ns_b, m.ns_c) == (3.4445, -4.7750, 2.0315)
    m, h = O._muon_hyper(dict(O._AUX_ADAMW_DEFAULTS, use_muon=False))
    assert (h.kind, h.lr, h.beta1, h.beta2, h.eps, h.weight_decay) == (_lib.OPT_ADAMW, 1e-3, 0.9, 0.999, 1e-8, 1e-2)
    assert m.ns_steps == 0


def test_load_step_counts_without_step():
    """Muon entries carry no step: a parameter with a momentum_buffer has stepped (opt_steps times, 1 in a torch-written
    checkpoint), one without an entry has not; AdamW entries carry their own."""
    buf = torch.zeros(2, 2)
    entries = [{"momentum_buffer": buf}, {}, {"step": torch.tensor(3.0), "exp_avg": buf, "exp_avg_sq": buf}]
    assert O.load_step_counts(O._MUON, entries, [0, 0, 1], None, True) == (3, [1, 0, 3], None)
    assert O.load_step_counts(O._MUON, entries, [0, 0, 1], 3, True) == (3, [3, 0, 3], None)


class _Model(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = torch.nn.Conv2d(3, 8, 3)
        self.fc = torch.nn.Linear(8, 4)


def _aux_kw(model, n_muon_groups=1):
    mats = [model.conv.weight, model.fc.weight]
    rest = [model.conv.bias, model.fc.bias]
    groups = [dict(params=mats[k::n_muon_groups], use_muon=True) for k in range(n_muon_groups)]
    return {"params": groups + [dict(params=rest, use_muon=False)]}


def test_routing():
    """Up to 8 groups fused, 9 not; torch.optim.Muon fused; the classes that have no fused step stay on the stock
    route; a Muon parameter whose flat elements do not form its matrix stays on the stock route."""
    m = _Model()
    assert O.fused_supported(MuonWithAuxAdamW, _aux_kw(m), m)
    kw = _aux_kw(m)
    kw["params"] = [dict(params=[p], use_muon=p.ndim > 1) for p in m.parameters()]
    kw["params"] += [dict(params=[], use_muon=False)] * 4
    assert len(kw["params"]) == 8 and O.fused_supported(MuonWithAuxAdamW, kw, m)
    kw["params"] += [dict(params=[], use_muon=False)]
    assert not O.fused_supported(MuonWithAuxAdamW, kw, m)
    if hasattr(torch.optim, "Muon"):
        lin = torch.nn.Sequential(torch.nn.Linear(4, 6, bias=False), torch.nn.Linear(6, 2, bias=False))
        assert O.fused_supported(torch.optim.Muon, {"lr": 0.02}, lin)
        assert O._KINDS[torch.optim.Muon] == O._MUON
    for cls, kw in ((torch.optim.RMSprop, {}), (torch.optim.Adagrad, {}), (torch.optim.Adam, {"amsgrad": True}),
                    (torch.optim.LBFGS, {}), (torch.optim.SparseAdam, {})):
        assert not O.fused_supported(cls, dict(kw, lr=1e-3), m)
    # a transposed view: dim 0 is not the outermost dim of the flat elements
    t = _Model()
    t.fc.weight = torch.nn.Parameter(torch.zeros(8, 4).T)
    assert not O.fused_supported(MuonWithAuxAdamW, _aux_kw(t), t)
    assert not O._muon_flat_matrix(t.fc.weight) and O._muon_flat_matrix(m.fc.weight)
    assert O._muon_flat_matrix(torch.zeros(8, 3, 3, 3).contiguous(memory_format=torch.channels_last))


def test_muon_kind_is_a_string_and_exported():
    import stoke_b200

    assert isinstance(O._KINDS[MuonWithAuxAdamW], str)
    assert "MuonWithAuxAdamW" in stoke_b200.__all__


def test_descriptor_table():
    """layout.muon_plan against the independent plan of tests/muon_ref.py: square, wide, tall (transposed), odd, 1 x n,
    n x 1 and a 30522 x 768 embedding-sized matrix, with non-Muon parameters between them."""
    shapes = [(64, 64), None, (768, 3072), (3072, 768), (33, 70), None, (1, 9), (9, 1), (30522, 768), (65, 129)]
    numels = [1 if s is None else s[0] * s[1] for s in shapes]
    offsets, _, _ = layout.param_offsets(numels)
    table, tot = layout.muon_plan(shapes, offsets)
    want = mr.plan(shapes)
    assert table == want
    last = want[-1]
    assert tot["tiles"] == last["tile0"] + -(-65 * 129 // 8192)
    assert tot["tri"] == last["tri0"] + 3 and tot["full"] == last["full0"] + 2 * 3
    assert tot["x_elems"] == last["x_offset"] + 65 * 129 + 7 and tot["a_elems"] == last["a_offset"] + 65 * 65 + 7
    assert [t["transposed"] for t in table] == [False, False, True, False, False, True, True, False]
    assert all(t["x_offset"] % 8 == 0 and t["a_offset"] % 8 == 0 and t["offset"] % 16 == 0 for t in table)


def test_c_structs():
    """stk_muon_param_t, stk_muon_hyper_t and stk_muon_args_t as include/stoke_b200.h lays them out (x86-64)."""
    assert C.sizeof(_lib.MuonParam) == 3 * 8 + 8 * 4 + 8
    assert _lib.MuonParam.lr_ratio.offset == 56
    assert C.sizeof(_lib.MuonHyper) == 7 * 8 + 2 * 4
    assert _lib.MuonArgs.params.offset == 32 and _lib.MuonArgs.param_group.offset == 56
    assert _lib.MuonArgs.lp_dtype.offset == 168 and C.sizeof(_lib.MuonArgs) == 176
    assert "stk_muon_step" in _lib.EXPORTS


def test_flop_count():
    """bench_muon.py's algorithmic FLOPs: ns_steps (4 r^2 c + 2 r^3) per matrix, r <= c."""
    import bench_muon

    assert bench_muon.ns_flops(768, 3072, 5) == mr.ns_flops(768, 3072, 5) == 5 * (4 * 768 ** 2 * 3072 + 2 * 768 ** 3)
    assert bench_muon.ns_flops(3072, 768, 5) == bench_muon.ns_flops(768, 3072, 5)
    assert bench_muon.ns_flops(1, 9, 2) == 2 * (4 * 9 + 2)
    bert = bench_muon.bert_base_matrices()
    assert len(bert) == 72 and bert.count((768, 768)) == 48 and bert.count((3072, 768)) == 12
    rn = bench_muon.resnet50_matrices()
    assert len(rn) == 53 and (64, 3 * 7 * 7) in rn and sum(r * c for r, c in rn) == 23454912
