# -*- coding: utf-8 -*-
"""CPU: stoke_b200.AdamW8bit / Adam8bit (bitsandbytes' 8-bit AdamW with block-wise quantized moments) against an
independent numpy transcription of its update (fp32, the same order of ops, the nearest code by a full scan of the map),
plus the maps, the quantization bound, argument validation, the state layout, step-count loading, routing, the ABI
structs and a tracking test against torch.optim.AdamW."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

import stoke_b200 as sb
from stoke_b200 import _lib
from stoke_b200.optim import (_STATE_LAYOUT, Adam8bit, AdamW8bit, check_8bit_entries, create_dynamic_map,
                              dequantize_blockwise, export_state, fused_supported, import_state, load_step_counts,
                              quantize_blockwise, state_buffers, state_dict_index)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32


# ---- the numpy transcription ---------------------------------------------------------------------------------------------
def np_quant(x, q):
    """codes, absmax of a 1-D fp32 array: n clamped into [q[0], q[255]], then the nearest map entry by a full scan (fp32
    |n - q|, first minimum)."""
    n = x.size
    nb = -(-n // 256)
    absmax = np.zeros(nb, f32)
    codes = np.zeros(n, np.uint8)
    for b in range(nb):
        blk = x[256 * b: 256 * (b + 1)]
        a = f32(np.max(np.abs(blk))) if not np.isnan(blk).any() else f32(np.nan)
        absmax[b] = a
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            inv = f32(0) if a == 0 else f32(f32(1) / a)
            y = (blk * inv).astype(f32)
        y[np.isnan(y)] = 0
        y = np.clip(y, q[0], q[-1])
        d = np.abs((y[:, None] - q[None, :]).astype(f32))
        codes[256 * b: 256 * (b + 1)] = np.argmin(d, axis=1)
    return codes, absmax


def np_deq(codes, q, absmax):
    with np.errstate(invalid="ignore"):
        return (q[codes.astype(np.int64)] * np.repeat(absmax, 256)[: codes.size]).astype(f32)


def np_step(w, g, st, hp, quant, q1, q2):
    """One step of one parameter on memory-ordered fp32 arrays; st: dict of numpy state, updated in place."""
    b1, b2 = hp["betas"]
    lr, eps, wd = hp["lr"], hp["eps"], hp["weight_decay"]
    st["step"] += 1
    t = float(st["step"])
    c1, c2 = 1 - b1 ** t, math.sqrt(1 - b2 ** t)
    if quant:
        m, v = np_deq(st["state1"], q1, st["absmax1"]), np_deq(st["state2"], q2, st["absmax2"])
    else:
        m, v = st["state1"], st["state2"]
    with np.errstate(invalid="ignore", over="ignore"):
        m = (m * f32(b1) + g * f32(1 - b1)).astype(f32)
        v = (v * f32(b2) + (g * g).astype(f32) * f32(1 - b2)).astype(f32)
        if wd != 0:
            w = (w * f32(1 - lr * wd)).astype(f32)
        den = (np.sqrt(v) + f32(eps * c2)).astype(f32)
        w = (w - (m / den).astype(f32) * f32(lr * c2 / c1)).astype(f32)
    if quant:
        st["state1"], st["absmax1"] = np_quant(m, q1)
        st["state2"], st["absmax2"] = np_quant(v, q2)
    else:
        st["state1"], st["state2"] = m, v
    return w


def mem(t):
    """A tensor's elements in memory order, as numpy."""
    x = t.detach().permute(sorted(range(t.dim()), key=lambda d: -t.stride(d)))
    return x.contiguous().view(-1).numpy().copy()


MIN = 128
SHAPES = [(127,), (128,), (129,), (300,), (16, 4, 3, 3), (40, 20), (7,)]   # below / at / above MIN, a short last block
CHANNELS_LAST = 4
NO_GRAD = 6          # never receives a gradient
ZERO_GRAD = 2        # a zero gradient at the first step: an all-zero block


def _params():
    g = torch.Generator().manual_seed(0)
    out = []
    for i, s in enumerate(SHAPES):
        p = torch.randn(*s, generator=g)
        if i == CHANNELS_LAST:
            p = p.to(memory_format=torch.channels_last)
        out.append(torch.nn.Parameter(p))
    return out


def _run(steps, nonfinite_at=None, cls=AdamW8bit):
    params = _params()
    groups = [dict(params=params[:4], lr=1e-2, weight_decay=0.1), dict(params=params[4:], lr=3e-3, betas=(0.8, 0.99))]
    opt = cls(groups, min_8bit_size=MIN)
    q1, q2 = create_dynamic_map(True).numpy(), create_dynamic_map(False).numpy()
    ref_w = [mem(p) for p in params]
    ref_st = [None] * len(params)
    gen = torch.Generator().manual_seed(1)
    for k in range(steps):
        for i, p in enumerate(params):
            g = torch.randn(p.shape, generator=gen).to(memory_format=torch.channels_last if i == CHANNELS_LAST else
                                                       torch.contiguous_format)
            if i == ZERO_GRAD and k == 0:
                g.zero_()
            if nonfinite_at is not None and k == nonfinite_at and i == 3:
                g.view(-1)[5] = float("nan")
                g.view(-1)[260] = float("inf")
            p.grad = None if i == NO_GRAD else g
        opt.step()
        for i, p in enumerate(params):
            if i == NO_GRAD:
                continue
            hp = opt.param_groups[0 if i < 4 else 1]
            quant = p.numel() >= MIN
            if ref_st[i] is None:
                n, nb = p.numel(), -(-p.numel() // 256)
                ref_st[i] = (dict(step=0, state1=np.zeros(n, np.uint8), state2=np.zeros(n, np.uint8),
                                  absmax1=np.zeros(nb, f32), absmax2=np.zeros(nb, f32)) if quant else
                             dict(step=0, state1=np.zeros(n, f32), state2=np.zeros(n, f32)))
            ref_w[i] = np_step(ref_w[i], mem(p.grad), ref_st[i], hp, quant, q1, q2)
    return params, opt, ref_w, ref_st


def _assert_matches(params, opt, ref_w, ref_st):
    for i, p in enumerate(params):
        if i == NO_GRAD:
            assert p not in opt.state or not opt.state[p]
            continue
        st = opt.state[p]
        np.testing.assert_array_equal(mem(p), ref_w[i], err_msg=f"weights {i}")
        assert float(st["step"]) == ref_st[i]["step"]
        for key in ("state1", "state2"):
            np.testing.assert_array_equal(mem(st[key]), ref_st[i][key], err_msg=f"{key} {i}")
            assert st[key].shape == p.shape and st[key].stride() == p.stride()
        if p.numel() >= MIN:
            assert st["state1"].dtype == torch.uint8
            for key in ("absmax1", "absmax2"):
                np.testing.assert_array_equal(st[key].numpy(), ref_st[i][key], err_msg=f"{key} {i}")
        else:
            assert st["state1"].dtype == torch.float32 and "qmap1" not in st and "absmax1" not in st


def test_class_against_numpy_transcription():
    params, opt, ref_w, ref_st = _run(5)
    _assert_matches(params, opt, ref_w, ref_st)
    # the all-zero block of the first step had absmax 0 and every code at the entry nearest 0
    assert list(opt.state[params[0]]) == ["step", "state1", "state2"]
    assert list(opt.state[params[1]]) == ["step", "state1", "qmap1", "state2", "qmap2", "absmax1", "absmax2"]


def test_all_zero_block_first_step():
    params, opt, ref_w, ref_st = _run(1)
    _assert_matches(params, opt, ref_w, ref_st)
    st = opt.state[params[ZERO_GRAD]]
    assert torch.equal(st["absmax1"], torch.zeros(1)) and torch.equal(st["absmax2"], torch.zeros(1))
    assert bool((st["state1"] == 127).all()) and bool((st["state2"] == 0).all())   # the codes of 0


def test_nonfinite_rule():
    params, opt, ref_w, ref_st = _run(4, nonfinite_at=2)
    _assert_matches(params, opt, ref_w, ref_st)
    st = opt.state[params[3]]   # 300 elements: block 0 held the NaN (and then decodes to NaN), block 1 the inf
    assert math.isnan(float(st["absmax1"][0])) and math.isnan(float(st["absmax1"][1]))
    w = params[3].detach()
    assert bool(torch.isnan(w.view(-1)[:256]).all())


def test_adam8bit_defaults():
    p = torch.nn.Parameter(torch.randn(300))
    assert Adam8bit([p]).defaults["weight_decay"] == 0.0 and AdamW8bit([p]).defaults["weight_decay"] == 1e-2
    params, opt, ref_w, ref_st = _run(3, cls=Adam8bit)
    _assert_matches(params, opt, ref_w, ref_st)


def test_maps():
    for signed in (True, False):
        q = create_dynamic_map(signed)
        assert q.dtype == torch.float32 and q.numel() == 256
        assert bool((q[1:] > q[:-1]).all()) and int((q == 0).sum()) == 1 and float(q.max()) == 1.0
    assert abs(float(create_dynamic_map(True)[0]) + 0.99297) < 1e-5 and float(create_dynamic_map(False)[0]) == 0.0


@pytest.mark.parametrize("signed", [True, False])
def test_round_trip_bound(signed):
    g = torch.Generator().manual_seed(3)
    x = torch.randn(256 * 7 + 13, generator=g) * torch.logspace(-6, 2, 256 * 7 + 13)
    x = x if signed else x.abs()
    q = create_dynamic_map(signed)
    code, absmax = quantize_blockwise(x, q)
    y = dequantize_blockwise(code, q, absmax)
    gaps = torch.cat([q[1:] - q[:-1], torch.zeros(1)])
    half = torch.maximum(gaps, torch.cat([torch.zeros(1), gaps[:-1]]))[code.long()] / 2
    a = absmax.repeat_interleave(256)[: x.numel()]
    assert bool(((y - x).abs() <= a * half * (1 + 1e-5) + 1e-30).all())


def _subnormal_blocks():
    """The subnormal-absmax blocks of optim8bit_edges_ref, one per 256-element block (zero-padded): as m, and as the v of
    the small gradients at beta2 = 0 and at the default beta2."""
    import optim8bit_edges_ref as er

    def pad(b):
        return np.pad(b, (0, 256 - b.size))

    m = np.concatenate([pad(er.subnormal_block(a)) for _, a in er.SUBNORMAL_ABSMAX])
    g0, g1 = er.v_subnormal_grads(4e-20), er.v_subnormal_grads(1e-18)
    v = np.concatenate([pad((g0 * g0).astype(f32)), pad(((g1 * g1).astype(f32) * f32(1 - 0.999)).astype(f32))])
    return m, v


def test_quantizer_edges_agree():
    """The class's quantize_blockwise, np_quant above and optim8bit_edges_ref.nearest_code give the same code for every
    crafted value: each default map's entries, its exact fp32 ties and their neighbours (in blocks of absmax 1, so n is
    the value), and blocks whose absmax is subnormal, where 1 / absmax overflows and n is +-inf: a positive element
    takes code 255, a negative one code 0, a zero the code of 0.  Under the default maps the clamp changes no code for a
    finite n, and the tie-to-upper mutant differs from the rule on the tie elements (150 of qmap1's gaps hold an exact
    fp32 tie, 92 of qmap2's one reachable as an fp32 square)."""
    import optim8bit_edges_ref as er

    q1, q2 = create_dynamic_map(True).numpy(), create_dynamic_map(False).numpy()
    assert er.nearest_code([np.inf, -np.inf, np.nan], q1).tolist() == [255, 0, 127]
    assert er.nearest_code([np.inf, -np.inf, np.nan], q2).tolist() == [255, 0, 0]
    rng = np.random.default_rng(11)
    x1 = er.blocks_with_unit_max(er.qmap1_values(q1), rng)
    g2 = er.blocks_with_unit_max(er.signed_shuffle(er.qmap2_values(q2), rng), rng)
    x2 = (g2 * g2).astype(f32)
    sub_m, sub_v = _subnormal_blocks()
    for q, x, sub, ties in ((q1, x1, sub_m, 150), (q2, x2, sub_v, 90)):
        for blocks in (x, sub):
            want, want_absmax = er.block_codes(blocks, q)
            code, absmax = quantize_blockwise(torch.from_numpy(blocks), torch.from_numpy(q))
            np_code, np_absmax = np_quant(blocks, q)
            np.testing.assert_array_equal(code.numpy(), want)
            np.testing.assert_array_equal(np_code, want)
            np.testing.assert_array_equal(absmax.numpy(), want_absmax)
            np.testing.assert_array_equal(np_absmax, want_absmax)
        assert (np.abs(x.reshape(-1, 256)).max(1) == 1).all()   # absmax 1: n is the value itself
        # the subnormal blocks: n = +-inf wherever 1 / absmax overflows
        absmax = quantize_blockwise(torch.from_numpy(sub), torch.from_numpy(q))[1].numpy()
        inf = np.repeat(er.overflows(absmax), 256)
        assert inf.sum() >= 256 * (3 if q is q1 else 2)
        code = quantize_blockwise(torch.from_numpy(sub), torch.from_numpy(q))[0].numpy()
        zero = int(er.nearest_code([0.0], q)[0])
        assert (code[inf & (sub > 0)] == 255).all() and (code[inf & (sub < 0)] == 0).all()
        assert (code[inf & (sub == 0)] == zero).all() and (inf & (sub > 0)).any()
        # the clamp changes nothing for a finite n under the default maps
        lo = -1.0 if q is q1 else 0.0
        y = np.concatenate([x, rng.uniform(lo, 1.0, 500_000).astype(f32),
                            np.array([np.nextafter(f32(1), f32(2)), f32(1.5), f32(lo - 0.5)], f32)])
        np.testing.assert_array_equal(er.nearest_code(y, q, clamp=False), er.nearest_code(y, q))
        # the tie rule is exercised
        assert int((er.nearest_code_upper(x, q) != er.nearest_code(x, q)).sum()) >= ties


@pytest.mark.parametrize("kw, name", [(dict(amsgrad=True), "amsgrad"), (dict(percentile_clipping=5), "percentile_clipping"),
                                      (dict(block_wise=False), "block_wise"), (dict(is_paged=True), "is_paged"),
                                      (dict(args=object()), "args")])
def test_refused_options(kw, name):
    with pytest.raises(ValueError, match=name):
        AdamW8bit([torch.nn.Parameter(torch.zeros(4))], **kw)


def test_accepted_options():
    p = torch.nn.Parameter(torch.zeros(4))
    AdamW8bit([p], optim_bits=8)
    for kw in (dict(lr=-1.0), dict(eps=-1.0), dict(betas=(1.0, 0.9)), dict(weight_decay=-0.1)):
        with pytest.raises(ValueError):
            AdamW8bit([p], **kw)


def _views_of(params, sd, min_size=MIN):
    """The fused step's views for these parameters, built on CPU tensors like GradPath's."""
    out = {t.key: [] for t in _STATE_LAYOUT["adam8bit"].tensors}
    q1, q2 = create_dynamic_map(True), create_dynamic_map(False)
    for p in params:
        if p.numel() >= min_size:
            nb = -(-p.numel() // 256)
            d = dict(state1=torch.zeros_like(p, dtype=torch.uint8), qmap1=q1, state2=torch.zeros_like(p, dtype=torch.uint8),
                     qmap2=q2, absmax1=torch.zeros(nb), absmax2=torch.zeros(nb))
        else:
            d = dict(state1=torch.zeros_like(p), state2=torch.zeros_like(p))
        for k in out:
            out[k].append(d.get(k))
    return out


def test_state_layout_round_trip():
    lay = _STATE_LAYOUT["adam8bit"]
    assert state_buffers(lay, [{}]) == {"M": None, "V": None, "M2": None}   # no fp32 moment buffers
    params, opt, _, _ = _run(3)
    sd = opt.state_dict()
    group_of = [0] * 4 + [1] * 3
    sd_index = state_dict_index(group_of, 2)
    entries = [sd["state"].get(sd_index[i], {}) for i in range(len(params))]
    views = _views_of(params, sd)
    import_state(lay, entries, views)
    steps = [0 if i == NO_GRAD else 3 for i in range(len(params))]
    state = export_state(lay, sd["param_groups"], group_of, sd_index, steps, None, views)
    assert set(state) == {sd_index[i] for i in range(len(params)) if i != NO_GRAD}
    for i in range(len(params)):
        if i == NO_GRAD:
            continue
        want, got = sd["state"][sd_index[i]], state[sd_index[i]]
        assert list(got) == list(want)
        for k in want:
            assert got[k].dtype == want[k].dtype and torch.equal(got[k], want[k]), (i, k)


def test_load_checks_and_python_int_step():
    params, opt, _, _ = _run(2)
    sd = opt.state_dict()
    fresh = AdamW8bit([dict(params=_params()[:4], lr=1e-2), dict(params=_params()[4:], lr=3e-3)], min_8bit_size=MIN)
    sd2 = {"state": {k: {kk: (int(vv) if kk == "step" else vv) for kk, vv in v.items()} for k, v in sd["state"].items()},
           "param_groups": sd["param_groups"]}
    fresh.load_state_dict(sd2)
    for p in fresh.state:
        st = fresh.state[p]
        assert torch.is_tensor(st["step"]) and st["step"].dtype == torch.float32 and float(st["step"]) == 2
        assert st["state1"].dtype == (torch.uint8 if p.numel() >= MIN else torch.float32)
    entries = [sd["state"].get(i, {}) for i in range(len(params))]
    quantized = [p.numel() >= MIN for p in params]
    check_8bit_entries(entries, quantized)
    with pytest.raises(ValueError, match="state1"):          # fp32 state for an 8-bit parameter
        check_8bit_entries(entries, [True] * len(params))
    bad = [dict(e) for e in entries]
    bad[1]["qmap1"] = bad[1]["qmap1"].flip(0)
    with pytest.raises(ValueError, match="ascending"):
        check_8bit_entries(bad, quantized)
    bad = [dict(e) for e in entries]
    bad[1]["qmap2"] = bad[1]["qmap2"] * 0.5
    with pytest.raises(ValueError, match="differ"):
        check_8bit_entries(bad, quantized)
    with pytest.raises(ValueError):
        AdamW8bit(_params(), min_8bit_size=10 ** 6).load_state_dict(
            {"state": sd["state"], "param_groups": [dict(sd["param_groups"][0], params=list(range(7)), min_8bit_size=10 ** 6)]})


def test_step_counts_load():
    entries = [{"step": 3}, {"step": torch.tensor(3.0)}, {}]
    steps, per_param, scal = load_step_counts("adam8bit", entries, [0, 0, 0], None, True)
    assert steps == 3 and per_param == [3, 3, 0] and scal is None


def _model(n_groups):
    return torch.nn.Sequential(*[torch.nn.Linear(4, 4) for _ in range(n_groups)])


@pytest.mark.parametrize("cls", [AdamW8bit, Adam8bit])
def test_routing(cls):
    for n, fused in ((8, True), (9, False)):
        m = _model(n)
        kw = dict(params=[dict(params=list(layer.parameters())) for layer in m], lr=1e-3)
        assert fused_supported(cls, kw, m) is fused
    assert not fused_supported(cls, dict(lr=1e-3, amsgrad=True), _model(1))
    assert sb.AdamW8bit is AdamW8bit and sb.Adam8bit is Adam8bit and {"AdamW8bit", "Adam8bit"} <= set(sb.__all__)
    assert _lib.Q8_BLOCK == 256


def test_abi_structs_against_the_header():
    assert C.sizeof(_lib.Adam8bitParam) == 24 and C.sizeof(_lib.Adam8bitHyper) == 40
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    fields = [f for f, _ in _lib.Adam8bitArgs._fields_]
    src = "#include <stdio.h>\n#include <stddef.h>\n#include \"stoke_b200.h\"\nint main(void) {\n"
    src += 'printf("%zu %zu %zu", sizeof(stk_adam8bit_param_t), sizeof(stk_adam8bit_hyper_t), sizeof(stk_adam8bit_args_t));\n'
    src += "".join(f'printf(" %zu", offsetof(stk_adam8bit_args_t, {f}));\n' for f in fields)
    src += 'printf(" %d", STK_Q8_BLOCK); return 0; }\n'
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "probe.c"), "w") as fh:
            fh.write(src)
        subprocess.check_call([cc, "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "probe"),
                               os.path.join(d, "probe.c")])
        got = [int(x) for x in subprocess.check_output([os.path.join(d, "probe")]).split()]
    want = [C.sizeof(_lib.Adam8bitParam), C.sizeof(_lib.Adam8bitHyper), C.sizeof(_lib.Adam8bitArgs)]
    want += [getattr(_lib.Adam8bitArgs, f).offset for f in fields] + [_lib.Q8_BLOCK]
    assert got == want


def test_tracks_adamw():
    """A fixed least-squares problem: 200 steps of AdamW8bit stay within 5 % (relative, in the weights) of
    torch.optim.AdamW with the same hyper-parameters, and reach a comparable loss."""
    g = torch.Generator().manual_seed(5)
    A, x_true = torch.randn(512, 64, generator=g), torch.randn(64, 128, generator=g)
    B = A @ x_true
    ws = [torch.nn.Parameter(torch.zeros(64, 128)) for _ in range(2)]
    opts = [AdamW8bit([ws[0]], lr=1e-2, weight_decay=1e-4, min_8bit_size=4096),
            torch.optim.AdamW([ws[1]], lr=1e-2, weight_decay=1e-4)]
    for _ in range(200):
        for w, o in zip(ws, opts):
            o.zero_grad()
            loss = ((A @ w - B) ** 2).mean()
            loss.backward()
            o.step()
    rel = float((ws[0] - ws[1]).detach().norm() / ws[1].detach().norm())
    assert rel < 0.05, rel
    l8, l32 = (float(((A @ w.detach() - B) ** 2).mean()) for w in ws)
    assert l8 < 1.5 * l32 + 1e-3, (l8, l32)
