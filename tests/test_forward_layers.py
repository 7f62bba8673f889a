"""The U-Net forward pass (ddpo_b200/unet.py, ``UNet.prepare_context`` and ``UNet.forward``) launch by launch: every
distinct kernel configuration SD2-base and SD1 launch, at sampling (batch 16, no tape) and at training (batch 40, tape),
replayed on the CUDA library against a float64 torch reference fed the same bf16-rounded operands.  The configurations
come from tests/_forward_census.py, which records the forward's launches on the ``meta`` device, so a new call site in
unet.py gets a case here without this file changing.  The whole-model tests allow ~2e-2 relative L2 on eps, enough to
hide a defect confined to one layer; these checks are per launch and use the bounds of tests/_layer_check.py.

Per configuration:
- weights go through ``prep_weight`` / ``permute_geglu_bias`` as ``UNet.refresh_weights`` does; the reference uses the
  natural (Flax) layout, so the weight layout is checked too;
- every output sits in a guarded buffer whose outside must come back unchanged, and must be finite;
- at batch 16 and 40 the float64 reference covers samples {0, 1, B/2, B-1} (0 and 1 share a 128-row tile at 8x8);
- inputs are drawn per sample from the sample's seed, so bit-level checks can compare one sample across launches: a
  rerun gives the same bits (without the GEMM's slab statistics: asking for them must not change the output), samples 0
  and B-1 computed alone equal their rows of the batch, and a sample gives the same bits at the other batch size of the
  forward (16 <-> 40) with the train pass's extra outputs (attention ``lse``, GEGLU ``aux_bf16``) toggled -- the PPO
  ratio of an unchanged policy is exactly 1 only if sampling and training agree bit for bit.

The TINY configurations replay on the torch-CPU emulation of the ops (value checks only) in the CPU suite.  The replays
of the ops the VAE launches too (igemm, GroupNorm, conv_in, cast_bf16, upsample2x_bf16) are in tests/_forward_replays.py.
"""
import math

import pytest
import torch
import torch.nn.functional as F
import _forward_census as census_mod
from _forward_replays import (_bit_checks, _check_vs_f32, _conv_ref, _designed, _finite, _gn_launch, _gn_ref,
                              _produce_unit, _rows, _seeded, _sel, _torch_f32_error, replay_cast_bf16,
                              replay_conv_in, replay_groupnorm_fwd, replay_igemm, replay_upsample2x_bf16)
from _layer_check import (BF16, BF16_L2, BF16_MAX, F32, F32_L2, F32_MAX, F32_ULP, F64, SINCOS_ARG_ULPS, SINCOS_ULPS,
                          Backend, Guarded, _current_node, _record, check_close, check_sum)  # noqa: F401


# ------------------------------------------------------------------------------------------------- norms ------
def _ln_ref(x, sc, bi):
    xd = x.double()
    mean = xd.mean(-1, keepdim=True)
    var = ((xd - mean) ** 2).mean(-1, keepdim=True)
    rstd = torch.rsqrt(var + 1e-5)
    return (xd - mean) * rstd * sc.double() + bi.double(), mean[:, 0], rstd[:, 0]


def _ln_launch(be, x, sc, bi, with_stats):
    m, c = x.shape
    y = Guarded(m, c, BF16, be.dev)
    st = Guarded(m, 2, F32, be.dev) if with_stats else None
    be.ops.layernorm_fwd(x, sc, bi, y.view, m, c, stats=st.view if st else None)
    be.sync()
    y.check("y")
    _finite("y", y.view)
    if st is not None:
        st.check("stats")
    return {"y": y.view, **({"stats": st.view} if st else {})}


def replay_layernorm_fwd(be, call):
    a, b = call.args, call.batch
    m, c = a["m"], a["c"]
    per = m // b
    with_stats = a.get("stats") is not None
    g = torch.Generator().manual_seed(c)
    sc = (1.0 + 0.1 * torch.randn(c, generator=g)).to(be.dev)
    bi = (0.1 * torch.randn(c, generator=g)).to(be.dev)
    launch = lambda seeds, variant: _ln_launch(be, _designed(be, seeds, per, c, 17), sc, bi,
                                               with_stats and variant != "rerun")
    x = _designed(be, list(range(b)), per, c, 17)
    got = _ln_launch(be, x, sc, bi, with_stats)
    sel = _sel(b)
    xs = _rows(x, sel, per)
    y, mean, rstd = _ln_ref(xs, sc, bi)
    check_close("y", _rows(got["y"], sel, per), y, BF16_MAX, BF16_L2)
    if with_stats and not be.emulated:
        st = _rows(got["stats"], sel, per)
        check_sum("mean", st[:, 0], mean, xs.double().abs().mean(-1))
        check_close("rstd", st[:, 1], rstd, F32_MAX, F32_L2)
    _bit_checks(be, b, launch, per)


# --------------------------------------------------------------------------------------------- attention ------
def replay_attention_fwd(be, call):
    a, b = call.args, call.batch
    heads, nq, nk, d = a["heads"], a["nq"], a["nk"], a.get("head_dim", 64)
    q_t, k_t, v_t = a["q"], a["k"], a["v"]
    self_attn = q_t.buf == k_t.buf
    ldq, ldk, ldv, ldo = a["ldq"], a["ldk"], a["ldv"], a["ldo"]
    assert k_t.buf == v_t.buf and ldk == ldv
    hd_kw = {"head_dim": d} if "head_dim" in a else {}

    def launch(seeds, variant):
        bb = len(seeds)
        qbuf = _seeded(be, seeds, nq, ldq, 19, scale=1.5).to(BF16)
        if self_attn:
            kbuf, k_off = qbuf, k_t.offset
        else:
            kbuf, k_off = _seeded(be, seeds, nk, ldk, 23, scale=1.5).to(BF16), 0
        v_off = k_off + v_t.offset - k_t.offset
        out = Guarded(bb * nq, ldo, BF16, be.dev)
        want_lse = (a.get("lse") is not None) != (variant == "other")
        lse = Guarded(bb * heads, nq, F32, be.dev) if want_lse and variant != "rerun" else None
        be.ops.attention_fwd(qbuf, kbuf[:, k_off:], kbuf[:, v_off:], out.view, bb, heads, nq, nk, ldq, ldk, ldv, ldo,
                             lse=lse.view if lse else None, **hd_kw)
        be.sync()
        out.check("out")
        _finite("out", out.view)
        res = {"out": out.view}
        if lse is not None:
            lse.check("lse")
            _finite("lse", lse.view)
            res["lse"] = lse.view.reshape(bb, heads * nq)
        return res, qbuf, kbuf, k_off, v_off

    got, qbuf, kbuf, k_off, v_off = launch(list(range(b)), "main")
    pairs = [(s, h) for s in (0, b - 1) for h in range(heads)] + [(b // 2, (b // 2) % heads)]
    max_err = max_ref = sq_err = sq_ref = 0.0
    lse_err = []
    for s, h in pairs:
        hc = slice(h * d, (h + 1) * d)
        q = qbuf[s * nq:(s + 1) * nq, hc].double()
        kk = kbuf[s * nk:(s + 1) * nk, k_off + h * d:k_off + (h + 1) * d].double()
        v = kbuf[s * nk:(s + 1) * nk, v_off + h * d:v_off + (h + 1) * d].double()
        sc = q @ kk.t() * d ** -0.5
        ref = torch.softmax(sc, -1) @ v
        dlt = got["out"][s * nq:(s + 1) * nq, hc].double() - ref
        max_err, max_ref = max(max_err, dlt.abs().max().item()), max(max_ref, ref.abs().max().item())
        sq_err, sq_ref = sq_err + (dlt * dlt).sum().item(), sq_ref + (ref * ref).sum().item()
        if "lse" in got and not be.emulated:      # the emulation does not write lse
            lse_err.append((got["lse"][s, h * nq:(h + 1) * nq].double(), torch.logsumexp(sc, -1)))
    e_max, e_l2 = max_err / max_ref, (sq_err / sq_ref) ** 0.5
    _record("out", max=e_max, l2=e_l2)
    assert e_max <= BF16_MAX and e_l2 <= BF16_L2, f"out: max err {e_max:.3g} * max|ref|, relative L2 {e_l2:.3g}"
    if lse_err:
        check_close("lse", torch.cat([g_ for g_, _ in lse_err]), torch.cat([r for _, r in lse_err]), F32_MAX, F32_L2)
    _bit_checks(be, b, lambda seeds, variant: launch(seeds, variant)[0], nq)


# ---------------------------------------------------------------------------------------------- sums ------
def replay_conv_out(be, call):
    a, b = call.args, call.batch
    h, wd, cin, cout = a["h"], a["wd"], a["cin"], a["cout"]
    g = torch.Generator().manual_seed(43)
    w = (torch.randn(3, 3, cin, cout, generator=g) * (9 * cin) ** -0.5).to(be.dev)
    bias = (torch.randn(cout, generator=g) * 0.5).to(be.dev)

    def launch(seeds, variant):
        bb = len(seeds)
        x = F.silu(_designed(be, seeds, h * wd, cin, 47))
        y = Guarded(bb * cout * h, wd, F32, be.dev)
        be.ops.conv_out(x, w, bias, y.view.view(bb, cout, h, wd), bb, h, wd, cin, cout)
        be.sync()
        y.check("y")
        _finite("y", y.view)
        return {"y": y.view}, x

    got, x = launch(list(range(b)), "main")
    sel = _sel(b)
    xs = _rows(x, sel, h * wd).double().reshape(len(sel), h, wd, cin)
    wr = w.double().reshape(9 * cin, cout)
    nchw = lambda t: t.reshape(len(sel), h, wd, cout).permute(0, 3, 1, 2).reshape(-1, wd)
    ref = nchw(_conv_ref(xs, wr, 1, 9) + bias.double())
    terms = nchw(_conv_ref(xs.abs(), wr.abs(), 1, 9) + bias.double().abs())
    check_sum("y", _rows(got["y"], sel, cout * h), ref, terms)
    _bit_checks(be, b, lambda seeds, variant: launch(seeds, variant)[0], cout * h)


def replay_dense_small(be, call):
    a, b = call.args, call.batch
    k, n, silu_out = a["k"], a["n"], a.get("silu_out", False)
    assert not a.get("silu_in")
    g = torch.Generator().manual_seed(k + n)
    w = (torch.randn(k, n, generator=g) * k ** -0.5).to(be.dev)
    bias = (torch.randn(n, generator=g) * 0.5).to(be.dev)

    def launch(seeds, variant):
        x = _seeded(be, seeds, 1, k, 53)
        y = Guarded(len(seeds), n, F32, be.dev)
        be.ops.dense_small(x, w, bias, y.view, len(seeds), k, n, silu_out=silu_out)
        be.sync()
        y.check("y")
        _finite("y", y.view)
        return {"y": y.view}, x

    got, x = launch(list(range(b)), "main")
    pre = x.double() @ w.double() + bias.double()
    terms = x.double().abs() @ w.double().abs() + bias.double().abs()
    # SiLU: |silu'| <= 1.1, plus its own fp32 evaluation (a few ulp of the result, inside 1e-5 |y|)
    ref = F.silu(pre) if silu_out else pre
    check_sum("y", got["y"], ref, 1.1 * terms + ref.abs() if silu_out else terms)
    _bit_checks(be, b, lambda seeds, variant: launch(seeds, variant)[0], 1)


def replay_dense_small_grouped(be, call):
    a, b = call.args, call.batch
    k, entries = a["k"], call.group_table
    total_params = a["params_base"].shape[0]
    total_y = a["y_base"].shape[0]
    params = torch.zeros(total_params, device=be.dev)   # full size: the offsets lie past 2^31 bytes for SD2
    g = torch.Generator(device=be.dev).manual_seed(59)
    for w_off, b_off, _, n in entries:
        params[w_off:w_off + k * n] = torch.randn(k * n, generator=g, device=be.dev) * k ** -0.5
        params[b_off:b_off + n] = torch.randn(n, generator=g, device=be.dev) * 0.5

    def launch(seeds, variant):
        bb = len(seeds)
        # the table holds each group's output offset for one batch size (UNet keeps one table per batch size)
        offs = [0]
        for *_, n in entries:
            offs.append(offs[-1] + bb * n)
        tab = [(w_off, b_off, y_off, n) for (w_off, b_off, _, n), y_off in zip(entries, offs)]
        assert bb != b or tab == entries
        table, ctas = be.ops.dense_small_group_table(tab, be.dev)
        x = F.silu(_seeded(be, seeds, 1, k, 61))
        y = Guarded(1, sum(bb * n for *_, n in entries), F32, be.dev)
        be.ops.dense_small_grouped(x, params, y.view[0], table, len(entries), ctas, bb, k)
        be.sync()
        y.check("y")
        _finite("y", y.view)
        # per sample: its row of every group's [B, n] block, in group order
        parts, off = [], 0
        for *_, n in entries:
            parts.append(y.view[0, off:off + bb * n].reshape(bb, n))
            off += bb * n
        return {"y": torch.cat(parts, 1)}, x

    assert total_y == sum(b * n for *_, n in entries)
    got, x = launch(list(range(b)), "main")
    refs, terms = [], []
    for w_off, b_off, _, n in entries:
        w = params[w_off:w_off + k * n].double().reshape(k, n)
        bias = params[b_off:b_off + n].double()
        refs.append(x.double() @ w + bias)
        terms.append(x.double().abs() @ w.abs() + bias.abs())
    check_sum("y", got["y"], torch.cat(refs, 1), torch.cat(terms, 1))
    _bit_checks(be, b, lambda seeds, variant: launch(seeds, variant)[0], 1)
    del params


TIMESTEPS = (0, 1, 21, 441, 981, 999)


def replay_timestep_sincos(be, call):
    from oracle.unet import timestep_embedding
    a, b = call.args, call.batch
    dim = a["dim"]
    half = dim // 2
    per_sample = torch.tensor([TIMESTEPS[i % len(TIMESTEPS)] for i in range(b)], dtype=torch.int32)
    cases = [(per_sample, per_sample)] + [(torch.tensor([t], dtype=torch.int32), torch.full((b,), t)) for t in TIMESTEPS]
    for t, t_full in cases:
        out = Guarded(b, dim, F32, be.dev)
        be.ops.timestep_sincos(t.to(be.dev), out.view, b, dim)
        be.sync()
        out.check("sincos")
        # float64 of the oracle's formula; the kernel's t * freq carries the fp32 rounding of freq and of the product
        inc = math.log(10000.0) / half
        arg = t_full.double()[:, None] * torch.exp(torch.arange(half, dtype=F64) * -inc)[None]
        ref = torch.cat([torch.cos(arg), torch.sin(arg)], 1)
        bound = torch.cat([arg, arg], 1) * (SINCOS_ARG_ULPS * F32_ULP) + SINCOS_ULPS * F32_ULP
        err = (out.view.cpu().double() - ref).abs()
        _record("sincos", worst_over_bound=(err / bound).max().item())
        assert (err <= bound).all(), f"timestep_sincos: error {(err / bound).max().item():.3g} x the bound"
        # the float64 formula is the oracle's (which computes in fp32)
        assert ((timestep_embedding(t_full, dim, torch.float32).double() - ref).abs() <= bound).all()


REPLAY = {"igemm": replay_igemm, "groupnorm_fwd": replay_groupnorm_fwd, "layernorm_fwd": replay_layernorm_fwd,
          "attention_fwd": replay_attention_fwd, "cast_bf16": replay_cast_bf16,
          "upsample2x_bf16": replay_upsample2x_bf16, "conv_in": replay_conv_in, "conv_out": replay_conv_out,
          "dense_small": replay_dense_small, "dense_small_grouped": replay_dense_small_grouped,
          "timestep_sincos": replay_timestep_sincos}


# ------------------------------------------------------------------------------------------ the census ------
def test_census_records_both_phases_of_every_run():
    for which in ("full", "tiny"):
        for run, (ctx_calls, fwd_calls) in census_mod.runs(which).items():
            ctx_ops = [c.op for c in ctx_calls]
            assert ctx_ops[0] == "cast_bf16" and set(ctx_ops[1:]) == {"igemm"}, (run, ctx_ops)
            fwd_ops = [c.op for c in fwd_calls]
            assert fwd_ops[0] == "timestep_sincos" and fwd_ops[-1] == "conv_out", run
            taped = run[2]
            assert all((c.args.get("lse") is not None) == taped for c in fwd_calls if c.op == "attention_fwd"), run
            assert all((c.args.get("aux_bf16") is not None) == taped for c in fwd_calls if c.args.get("geglu")), run


def test_every_recorded_op_has_a_replay():
    ops = {c.op for which in ("full", "tiny") for _, c, _ in census_mod.census(which)}
    missing = ops - set(REPLAY)
    assert not missing, f"forward ops without a replay in test_forward_layers.py: {sorted(missing)}"


def test_each_signature_has_one_test_id():
    for which in ("full", "tiny"):
        entries = census_mod.census(which)
        assert len({k for k, _, _ in entries}) == len(entries)
        ids = [c.test_id() for _, c, _ in entries]
        assert len(set(ids)) == len(ids), which


def _census_params():
    out = [pytest.param("emulator", c, id="emu-" + c.test_id()) for _, c, _ in census_mod.census("tiny")]
    out += [pytest.param("cuda", c, marks=pytest.mark.gpu, id="cuda-" + c.test_id())
            for _, c, _ in census_mod.census("full")]
    return out


@pytest.mark.parametrize("backend,call", _census_params())
def test_forward_launch(backend, call):
    torch.backends.cuda.matmul.allow_tf32 = False
    be = Backend(backend)
    REPLAY[call.op](be, call)


# ----------------------------------------------------------------------- norms fed a residual with a DC offset ------
DC_MU = (0, 8, 64)


@pytest.mark.gpu
@pytest.mark.parametrize("mu", DC_MU)
@pytest.mark.parametrize("b,hw,c", [(4, 4096, 320), (16, 64, 1280)])
def test_groupnorm_dc_offset(b, hw, c, mu):
    """GroupNorm of a stream tensor whose groups sit at an offset of mu standard deviations: the statistics are
    E[x^2] - E[x]^2 in fp32, from the slab sums of the producing GEMM and from the two-pass path"""
    be = Backend("cuda")
    seeds = list(range(b))
    # per-group offset mu * sigma (sigma ~ 1 by construction of the residual around 0), signs alternating by group
    g = torch.Generator().manual_seed(67)
    per_group = mu * torch.where(torch.arange(32) % 2 == 0, 1.0, -1.0) * (1 + 0.1 * torch.rand(32, generator=g))
    dc = per_group.repeat_interleave(c // 32).to(be.dev)
    x, st = _produce_unit(be, seeds, hw, c, dc)
    sc = torch.ones(c, device=be.dev)
    bi = torch.zeros(c, device=be.dev)
    ref_fn = lambda v: _gn_ref(v, sc, bi, b, hw, False)

    def f32_fn(v):
        t = v.reshape(b, hw, 32, c // 32)
        mean = t.mean(dim=(1, 3), keepdim=True)
        var = ((t * t).mean(dim=(1, 3), keepdim=True) - mean * mean).clamp(min=0)
        return ((t - mean) * torch.rsqrt(var + 1e-5)).reshape(-1, c)

    e32 = _torch_f32_error(x, ref_fn, f32_fn)
    ref = ref_fn(x)
    for name, s0 in (("slab stats", st), ("two-pass", None)):
        got = _gn_launch(be, x, None, s0, None, sc, bi, b, hw, c, 0, False, ["y_f32", "y_bf16"])
        _check_vs_f32(name + " y_f32", got["y_f32"], ref, e32, F32_MAX, F32_L2)
        _check_vs_f32(name + " y_bf16", got["y_bf16"], ref, e32, BF16_MAX, BF16_L2)




@pytest.mark.gpu
@pytest.mark.parametrize("mu", DC_MU)
@pytest.mark.parametrize("m,c", [(4 * 4096, 320), (16 * 64, 1280)])
def test_layernorm_dc_offset(m, c, mu):
    """LayerNorm of rows offset by mu standard deviations (each row its own offset, of either sign)"""
    be = Backend("cuda")
    g = torch.Generator(device="cuda").manual_seed(73)
    dc = mu * (1 + 0.1 * torch.rand(m, 1, generator=g, device="cuda")) * torch.where(
        torch.arange(m, device="cuda")[:, None] % 2 == 0, 1.0, -1.0)
    x = torch.randn(m, c, generator=g, device="cuda") + dc
    sc = torch.ones(c, device="cuda")
    bi = torch.zeros(c, device="cuda")

    def f32_fn(v):
        mean = v.mean(-1, keepdim=True)
        var = ((v * v).mean(-1, keepdim=True) - mean * mean).clamp(min=0)
        return (v - mean) * torch.rsqrt(var + 1e-5)

    e32 = _torch_f32_error(x, lambda v: _ln_ref(v, sc, bi)[0], f32_fn)
    got = _ln_launch(be, x, sc, bi, True)
    y, _, rstd = _ln_ref(x, sc, bi)
    _check_vs_f32("y", got["y"], y, e32, BF16_MAX, BF16_L2)
    e32r = _torch_f32_error(x, lambda v: _ln_ref(v, sc, bi)[2],
                            lambda v: torch.rsqrt((v * v).mean(-1) - v.mean(-1) ** 2 + 1e-5))
    _check_vs_f32("rstd", got["stats"][:, 1], rstd, e32r, F32_MAX, F32_L2)
