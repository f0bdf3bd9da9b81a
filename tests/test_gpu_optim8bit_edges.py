"""The fused 8-bit AdamW step (``stk_adam8bit_step``) at the quantizer's edges (GPU).

Every case runs the fused step and the class's ``step()`` on CUDA fp32 tensors from the same weights and compares them
bit for bit after every step -- master, codes, absmax, the fp32 state of the small parameters and the step counts -- on
the fp32 model's raw route, where the kernel receives the gradient exactly (bf16 only for the inf gradient):

  ties         betas (0, 0), so m = g and v = fp32(g * g), on blocks of absmax 1 whose elements are the maps' entries,
               their exact fp32 ties and neighbours (tests/optim8bit_edges_ref.py): the codes are also the reference's
               nearest codes, and the tie-to-upper mutant disagrees with the kernel on the tie elements
  overflow     blocks whose absmax is at or below 2 ** -128, where 1 / absmax is +inf and n = +-inf: code 255 for a
               positive element, 0 for a negative one, the code of 0 for a zero; then the default betas, so the decoded
               state reaches the master
  maps         a class checkpoint with a linear signed map and an unsigned map without 0 whose top entries are 0.25 and
               0.25 + 2 ** -25 (n = 1 is equally far from both in fp32), continued on crafted and random gradients
  tails        an all-zero block, parameters of 4096 + 13, 4096 + 255 and 8192 elements, a channels-last conv weight
               whose last block ends inside a lane; an inf gradient on the bf16 route, which makes its block decode to
               NaN at the next step
  scale        a 30522 x 768 embedding and 300 small parameters: at least three passes of the step's grid-stride loop
               and two CTAs of the prologue, with per-parameter skips"""
import numpy as np
import pytest
import torch

import optim8bit_edges_ref as er
from test_gpu_optim8bit import Shapes, _check, _fused, _reference, _same

pytestmark = pytest.mark.gpu

DEFAULT_BETAS = (0.9, 0.999)


def _maps():
    from stoke_b200.optim import create_dynamic_map

    return create_dynamic_map(True).numpy(), create_dynamic_map(False).numpy()


def _build(shapes, groups, lp=None):
    torch.cuda.set_device(0)
    net = Shapes(shapes).cuda()
    opt = _fused(net, lp, "local", groups=groups)
    ref, ropt = _reference(opt.path, groups=groups)
    return opt, ref, ropt


def _step(opt, ref, ropt, grads, tag, skip=()):
    """One fused step on ``grads`` (fp32 CUDA tensors shaped like the parameters) and one class step on the same, the
    parameters in ``skip`` without a gradient; then the bit-for-bit comparison."""
    path = opt.path
    for gv, g in zip(path.grad_views, grads):
        gv.copy_(g)
    path._track_touched = True
    path._touched = np.array([i not in skip for i in range(len(path.params))])
    path.after_backward(sync=True, unscale=False)
    opt.step()
    for i, (p, g) in enumerate(zip(ref, grads)):
        p.grad = None if i in skip else g.float()
    ropt.step()
    assert float(path.g_flat.float().abs().max()) == 0.0, tag   # the raw bucket is consumed
    _check(path, ref, ropt, tag)


def _cuda(x, shape=None):
    t = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).cuda()
    return t if shape is None else t.view(shape)


def _codes(opt, i, key):
    return opt.path.adam8bit_state_views()[i][key].detach().reshape(-1).cpu().numpy()


def _blocks(crafted, n_blocks, numel, rng):
    """``n_blocks`` blocks of absmax 1 (tests/optim8bit_edges_ref.py), the crafted ones at random places before the last
    block, the rest random in [-1, 1]; cut to ``numel`` elements."""
    crafted = crafted.reshape(-1, er.BLOCK)
    fill = er.blocks_with_unit_max(rng.uniform(-1, 1, (n_blocks - len(crafted)) * (er.BLOCK - 1)), rng)
    out = fill.reshape(-1, er.BLOCK)
    out = np.insert(out, np.sort(rng.integers(0, len(out), len(crafted))), crafted, axis=0)
    return out.reshape(-1)[:numel]


# ---- exact ties ---------------------------------------------------------------------------------------------------------
TIE_SHAPES = [((4096,), False), ((4352,), False), ((5000,), False), ((1000,), False)]


def test_ties_go_to_the_lower_code():
    q1, q2 = _maps()
    rng = np.random.default_rng(0)
    m_blocks = er.blocks_with_unit_max(er.qmap1_values(q1), rng)                          # n1 = g
    v_blocks = er.blocks_with_unit_max(er.signed_shuffle(er.qmap2_values(q2), rng), rng)  # n2 = fp32(g * g)
    crafted = np.concatenate([m_blocks, v_blocks]).reshape(-1, er.BLOCK)
    parts = np.array_split(np.arange(len(crafted)), 3)   # spread over the three quantized parameters
    grads = []
    for (shape, _), idx in zip(TIE_SHAPES[:3], parts):
        n = shape[0]
        grads.append(_blocks(crafted[idx], -(-n // er.BLOCK), n, rng))
    grads.append(rng.uniform(-1, 1, 1000).astype(np.float32))
    opt, ref, ropt = _build(TIE_SHAPES, [([0, 1, 2, 3], dict(betas=(0.0, 0.0)))])
    for step in range(2):
        _step(opt, ref, ropt, [_cuda(g) for g in grads], ("ties", step))
        ties = {"state1": 0, "state2": 0}
        for i, g in enumerate(grads[:3]):
            for key, n, q in (("state1", g, q1), ("state2", (g * g).astype(np.float32), q2)):
                got, want, upper = _codes(opt, i, key), er.nearest_code(n, q), er.nearest_code_upper(n, q)
                np.testing.assert_array_equal(got, want, err_msg=f"{key} of parameter {i}, step {step}")
                tie = want != upper
                assert (got[tie] != upper[tie]).all()
                ties[key] += int(tie.sum())
        assert ties["state1"] >= 150 and ties["state2"] >= 90, ties
    opt.close()


# ---- 1 / absmax overflows -----------------------------------------------------------------------------------------------
def _pad(b):
    return np.pad(b, (0, er.BLOCK - b.size))


def _assert_overflow_codes(opt, i, g, key, tag):
    """Where 1 / absmax overflowed: 255 for a positive element, 0 for a negative one, the code of 0 for a zero.  ``g``
    carries the element's sign (m has the gradient's sign; for v pass |g|: v is positive where g is nonzero).  Returns
    how many elements of overflowing blocks there were."""
    absmax = opt.path.adam8bit_state_views()[i]["absmax1" if key == "state1" else "absmax2"].cpu().numpy()
    inf = np.repeat(er.overflows(absmax), er.BLOCK)[: g.size]
    code = _codes(opt, i, key)
    q = _maps()[0 if key == "state1" else 1]
    want = np.where(g > 0, 255, np.where(g < 0, 0, er.nearest_code([0.0], q)[0]))
    bad = inf & (code != want)
    assert not bad.any(), (tag, key, i, "codes", code[bad][:16].tolist(), "expected", want[bad][:16].tolist())
    return int(inf.sum())


def test_overflowing_reciprocal():
    # parameter 0: m blocks of subnormal absmax (their v = g * g underflows to an all-zero block); parameter 1: v blocks
    # of g near 4e-20 (v = g * g at beta2 = 0); parameter 2 (default betas throughout): g near 1e-18, v = 1e-3 g * g
    rng = np.random.default_rng(1)
    sub_m = np.concatenate([_pad(er.subnormal_block(a)) for _, a in er.SUBNORMAL_ABSMAX])
    sub_v0 = np.concatenate([_pad(er.v_subnormal_grads(4e-20)), _pad(er.v_subnormal_grads(3e-20))])
    sub_v1 = np.concatenate([_pad(er.v_subnormal_grads(1e-18)), _pad(er.v_subnormal_grads(7e-19))])
    assert ((sub_v0 * sub_v0 != 0) == (sub_v0 != 0)).all()   # no square underflows: v > 0 exactly where g != 0
    assert (((sub_v1 * sub_v1).astype(np.float32) * np.float32(1 - 0.999) != 0) == (sub_v1 != 0)).all()
    fixed = [sub_m, sub_v0, sub_v1]
    shapes = [((4096,), False), ((4096,), False), ((4096,), False), ((700,), False)]
    groups = [([0, 1, 3], dict(betas=(0.0, 0.0))), ([2], dict(betas=DEFAULT_BETAS))]
    opt, ref, ropt = _build(shapes, groups)
    for step in range(4):
        if step == 1:   # the default betas from here on: the decoded state feeds m, v and the master
            for gr in (opt.param_groups[0], ropt.param_groups[0]):
                gr["betas"] = DEFAULT_BETAS
        grads = []
        for f in fixed:
            rest = (rng.standard_normal(4096 - f.size) * 1e-2).astype(np.float32)
            grads.append(np.concatenate([f, rest]))
        grads.append((rng.standard_normal(700) * 1e-2).astype(np.float32))
        path = opt.path
        for gv, g in zip(path.grad_views, grads):
            gv.copy_(_cuda(g))
        path.after_backward(sync=True, unscale=False)
        opt.step()
        # the literal codes first: without the clamp an n of +inf takes code 254
        n1 = _assert_overflow_codes(opt, 0, grads[0], "state1", step)
        n2 = _assert_overflow_codes(opt, 1, np.abs(grads[1]), "state2", step)
        n3 = _assert_overflow_codes(opt, 2, np.abs(grads[2]), "state2", step)
        assert n1 >= 3 * er.BLOCK and n2 >= 2 * er.BLOCK and n3 >= er.BLOCK, (step, n1, n2, n3)
        for p, g in zip(ref, grads):
            p.grad = _cuda(g)
        ropt.step()
        _check(path, ref, ropt, ("overflow", step))
    opt.close()


# ---- maps from a checkpoint ---------------------------------------------------------------------------------------------
def _other_maps():
    q1 = torch.linspace(-1, 1, 256, dtype=torch.float32)
    q2 = torch.linspace(2.0 ** -10, 0.25, 255, dtype=torch.float32)
    q2[-1] = 0.25
    q2 = torch.cat([q2, torch.tensor([0.25 + 2.0 ** -25])])
    assert float(q1[-1]) == 1.0 and float(q2[-1]) - float(q2[-2]) == 2.0 ** -25 and bool((q2[1:] > q2[:-1]).all())
    return q1, q2


def test_non_default_maps_from_a_checkpoint():
    shapes = [((4096,), False), ((4096 + 100,), False), ((1000,), False)]
    groups = [([0, 1, 2], {})]
    opt, ref, ropt = _build(shapes, groups)
    path = opt.path
    rng = np.random.default_rng(2)
    n0 = 5 * er.BLOCK   # parameter 0's first blocks: zero at the first step, then subnormal (n = +-inf under the maps)
    sub = np.concatenate([_pad(er.subnormal_block(a)) for _, a in er.SUBNORMAL_ABSMAX])
    for step in range(4):
        if step == 1:
            q1, q2 = _other_maps()
            sd = ropt.state_dict()
            state = {k: (dict(v, qmap1=q1.cuda(), qmap2=q2.cuda()) if "qmap1" in v else dict(v))
                     for k, v in sd["state"].items()}
            ck = {"state": state, "param_groups": sd["param_groups"]}
            ropt.load_state_dict(ck)
            opt.load_state_dict(ck)
            assert torch.equal(path.q8_qmap1.cpu(), q1) and torch.equal(path.q8_qmap2.cpu(), q2)
            _check(path, ref, ropt, "loaded")
        g0 = (rng.standard_normal(4096) * 1e-2).astype(np.float32)
        g0[:n0] = 0 if step == 0 else sub
        g1 = (rng.standard_normal(4196) * 1e-2).astype(np.float32)
        g2 = (rng.standard_normal(1000) * 1e-2).astype(np.float32)
        _step(opt, ref, ropt, [_cuda(g) for g in (g0, g1, g2)], ("maps", step))
        if step >= 1:
            assert bool((path.q8_code2 == 255).any()) and bool((path.q8_code1 == 255).any())
    opt.close()


# ---- non-finite gradients and tails -------------------------------------------------------------------------------------
TAIL_SHAPES = [((4096 + 13,), False), ((4096 + 255,), False), ((8192,), False), ((36, 13, 3, 3), True), ((333,), False)]


def test_zero_block_and_tails():
    assert 36 * 13 * 9 % er.BLOCK % 8 != 0   # the conv weight's last block ends inside a lane
    opt, ref, ropt = _build(TAIL_SHAPES, [([0, 2, 4], dict(weight_decay=0.01)), ([1, 3], dict(betas=(0.8, 0.99)))])
    g = torch.Generator(device="cuda").manual_seed(3)
    for step in range(4):
        grads = [torch.randn(p.shape, device="cuda", generator=g) * 1e-2 for p in ref]
        grads[3] = grads[3].contiguous(memory_format=torch.channels_last)
        if step == 0:
            grads[2].view(-1)[er.BLOCK: 2 * er.BLOCK] = 0   # an all-zero block at the first step
        _step(opt, ref, ropt, grads, ("tails", step))
        if step == 0:
            st = opt.path.adam8bit_state_views()[2]
            assert float(st["absmax1"][1]) == 0.0 and float(st["absmax2"][1]) == 0.0
            assert bool((st["state1"][er.BLOCK: 2 * er.BLOCK] == 127).all())
            assert bool((st["state2"][er.BLOCK: 2 * er.BLOCK] == 0).all())
    opt.close()


def test_inf_gradient_bf16_raw():
    """bf16 model, raw route, no loss scaler: an inf gradient makes its block's absmax inf, every element of the block
    takes the code of 0 (the finite ones have n = 0), and the block decodes to NaN at the next step."""
    shapes = [((4096 + 40,), False), ((1000,), False)]
    opt, ref, ropt = _build(shapes, [([0, 1], {})], lp=torch.bfloat16)
    path = opt.path
    g = torch.Generator(device="cuda").manual_seed(4)
    for step in range(3):
        grads = [(torch.randn(p.shape, device="cuda", generator=g) * 1e-2).bfloat16() for p in ref]
        if step == 1:
            grads[0][2 * er.BLOCK + 7] = float("inf")
        _step(opt, ref, ropt, grads, ("inf", step))
        st = path.adam8bit_state_views()[0]
        if step == 1:
            assert float(st["absmax1"][2]) == float("inf") and float(st["absmax2"][2]) == float("inf")
            assert bool((st["state1"][2 * er.BLOCK: 3 * er.BLOCK] == 127).all())
            assert bool((st["state2"][2 * er.BLOCK: 3 * er.BLOCK] == 0).all())
        if step == 2:
            w = path.unflatten(path.gather_master())[0]
            assert bool(torch.isnan(w[2 * er.BLOCK: 3 * er.BLOCK]).all()) and not bool(torch.isnan(w[: 2 * er.BLOCK]).any())
            assert torch.isnan(st["absmax1"][2]) and torch.isnan(st["absmax2"][2])
        assert _same(path.p_flat.float(), path.gather_master().to(torch.bfloat16).float())
    opt.close()


# ---- the grid-stride loop and the prologue's second CTA ----------------------------------------------------------------
def test_grid_stride_loop_and_prologue_ctas():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    small = [((7 + (i * 13) % 90,), False) for i in range(300)]
    shapes = [((30522, 768), False)] + small
    blocks = -(-30522 * 768 // er.BLOCK) + len(small)
    assert blocks >= 3 * 16 * sms * 8 and len(shapes) > 256, (blocks, sms)
    groups = [(list(range(0, len(shapes), 2)), dict(weight_decay=0.01)), (list(range(1, len(shapes), 2)), dict(lr=3e-3))]
    opt, ref, ropt = _build(shapes, groups)
    g = torch.Generator(device="cuda").manual_seed(5)
    skips = [(), (0,) + tuple(range(1, 301, 7)), tuple(range(2, 301, 5))]
    for step, skip in enumerate(skips):
        grads = [torch.randn(p.shape, device="cuda", generator=g) * 1e-2 for p in ref]
        _step(opt, ref, ropt, grads, ("scale", step), skip=set(skip))
        del grads
    assert opt.path.param_steps()[0] == 2 and opt.path.param_steps()[1] == 2
    opt.close()
