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

The TINY configurations replay on the torch-CPU emulation of the ops (value checks only) in the CPU suite.
"""
import math

import pytest
import torch
import torch.nn.functional as F
import _forward_census as census_mod
from _layer_check import (BF16, BF16_L2, BF16_MAX, F32, F32_L2, F32_MAX, F32_ULP, F64, NORM_DC_FACTOR, SINCOS_ARG_ULPS,
                          SINCOS_ULPS, Backend, Guarded, _current_node, _record, check_close, check_sum)  # noqa: F401

OTHER_BATCH = {16: 40, 40: 16}      # the forward's two batch sizes: sampling (2 x 8 for CFG) and the PPO train pass


# ----------------------------------------------------------------------------------------------- helpers ------
def _seeded(be, seeds, rows, cols, salt, scale=1.0, shift=0.0):
    """[len(seeds) * rows, cols] fp32: the block of a sample depends on its seed (and the operand's salt) only"""
    out = []
    for s in seeds:
        g = torch.Generator(device=be.dev).manual_seed(1_000_003 * salt + s)
        out.append(torch.randn(rows, cols, generator=g, device=be.dev) * scale + shift)
    return torch.cat(out)


def _sel(b):
    """samples the float64 reference covers"""
    return sorted({0, 1, b // 2, b - 1})


def _other_seeds(b):
    """seeds of the other-batch launch: B-1 and 0 at indices 0 and 1, fresh seeds after them"""
    b2 = OTHER_BATCH[b]
    return [b - 1, 0] + [10_000 + i for i in range(b2 - 2)]


def _rows(t, idx, per):
    """rows of samples ``idx`` in a [B * per, ...] tensor"""
    return torch.cat([t[i * per:(i + 1) * per] for i in idx])


def _finite(name, *ts):
    for t in ts:
        assert torch.isfinite(t.float()).all(), f"{name}: non-finite output"


def _same_bits(name, a, b):
    """bit equality (torch.equal would call -0.0 and 0.0 equal)"""
    as_int = lambda t: t.contiguous().view(torch.int16 if t.dtype == BF16 else torch.int32)
    assert a.shape == b.shape and torch.equal(as_int(a), as_int(b)), f"{name}: bits differ"


def _bit_checks(be, b, launch, per):
    """launch(seeds, variant) -> {name: [rows, ...] tensor, ``per`` rows per sample}; variant "main" as recorded, "rerun"
    without optional side outputs that must not change the main ones, "other" with the train pass's extra outputs toggled"""
    if be.emulated:
        return
    ref = launch(list(range(b)), "main")
    again = launch(list(range(b)), "rerun")
    for k in again:
        _same_bits(f"{k} rerun", again[k], ref[k])
    for s in (0, b - 1):
        alone = launch([s], "rerun")
        for k in alone:
            _same_bits(f"{k} of sample {s} alone", alone[k], ref[k][s * per:(s + 1) * per])
    if b in OTHER_BATCH:
        other = launch(_other_seeds(b), "other")
        for k in other:
            for i, s in enumerate((b - 1, 0)):
                if k in ref:
                    _same_bits(f"{k} of sample {s} at batch {OTHER_BATCH[b]}", other[k][i * per:(i + 1) * per],
                               ref[k][s * per:(s + 1) * per])


def _conv_ref(x, w, stride, taps):
    """float64 conv of NHWC x [S, Hi, Wi, Cin] with the natural kernel w [taps * Cin, N] ((ky, kx, cin) rows), padding 1
    for 3x3: one float64 GEMM per tap"""
    s, hi, wi, cin = x.shape
    n = w.shape[1]
    if taps == 1:
        return x.reshape(-1, cin) @ w
    ho, wo = hi // stride, wi // stride
    xp = F.pad(x, (0, 0, 1, 1, 1, 1))
    y = torch.zeros(s * ho * wo, n, dtype=x.dtype, device=x.device)
    for ky in range(3):
        for kx in range(3):
            patch = xp[:, ky:ky + stride * ho:stride, kx:kx + stride * wo:stride]
            y += patch.reshape(-1, cin) @ w[(ky * 3 + kx) * cin:(ky * 3 + kx + 1) * cin]
    return y


def _gelu_tanh(v):
    return 0.5 * v * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (v + 0.044715 * v ** 3)))


def _slab_check(name, st, y):
    """slab statistics [rows/32, n, 2] against float64 per-32-row sums of the kernel's own fp32 output y"""
    n = y.shape[1]
    t = y.double().reshape(-1, 32, n)
    check_sum(name + " sum", st[..., 0], t.sum(1), t.abs().sum(1))
    sq = (t * t).sum(1)
    check_sum(name + " sumsq", st[..., 1], sq, sq)


# -------------------------------------------------------------------------------------------------- igemm ------
def _weight_parts(a):
    """how many prep_weight calls UNet.refresh_weights makes for this GEMM's weight (q|k|v: 3, context k|v: 2)"""
    if a.get("conv") or a.get("bias") is not None or a.get("geglu"):
        return 1
    n, c0 = a["n"], a["c0"]
    return 3 if n == 3 * c0 else (1 if n == c0 else 2)


def replay_igemm(be, call):
    a, b = call.args, call.batch
    assert a.get("a1") is None and not a.get("accumulate") and not a.get("ld_out") and not a.get("lda0")
    conv, taps, stride, n, c0 = a.get("conv"), a.get("taps", 1), a.get("stride", 1), a["n"], a["c0"]
    geglu, has = bool(a.get("geglu")), (lambda k: a.get(k) is not None)
    per_out = conv[1] * conv[2] if conv else a["m"] // b
    per_in = per_out * stride * stride
    k = taps * c0
    g = torch.Generator().manual_seed(len(call.test_id()) * 7919 + n + k)
    w = torch.randn(k, n, generator=g) * k ** -0.5               # natural layout: Flax [kh, kw, cin, n] as [k, n]
    bias = torch.randn(n, generator=g) * 0.5 if has("bias") else None
    wt = torch.empty(n, k, dtype=BF16, device=be.dev)
    bias_arg = None
    if geglu:
        be.ops.prep_weight(w.to(be.dev), wt, k, n, geglu_bn=a["bn"])
        bias_arg = torch.empty(n, device=be.dev)
        be.ops.permute_geglu_bias(bias.to(be.dev), bias_arg, n, a["bn"])
    else:
        p = _weight_parts(a)
        for i in range(p):
            cols = slice(i * n // p, (i + 1) * n // p)
            be.ops.prep_weight(w[:, cols].contiguous().to(be.dev), wt, k, n // p, row_offset=i * n // p)
        bias_arg = bias.to(be.dev) if bias is not None else None
    n_out = n // 2 if geglu else n

    def launch(seeds, variant):
        bb = len(seeds)
        m = bb * per_out
        a0 = _seeded(be, seeds, per_in, c0, 1).to(BF16)
        rowvec = _seeded(be, seeds, 1, n, 2) if has("rowvec") else None
        res = _seeded(be, seeds, per_out, n, 3, scale=2.0, shift=1.0) if has("residual") else None
        outs = {}
        if has("out_f32"):
            outs["out_f32"] = Guarded(m, n, F32, be.dev)
        if has("out_bf16"):
            outs["out_bf16"] = Guarded(m, n_out, BF16, be.dev)
        if has("aux_bf16") != (variant == "other" and geglu):
            outs["aux_bf16"] = Guarded(m, n, BF16, be.dev)
        st = Guarded(-(-m // 32), 2 * n, F32, be.dev) if has("gn_stats") and variant == "main" else None
        kw = dict(conv=(bb, conv[1], conv[2])) if conv else dict(m=m)
        be.ops.igemm(a0=a0, wt=wt, n=n, c0=c0, taps=taps, stride=stride, bias=bias_arg, rowvec=rowvec,
                     rows_per_sample=a.get("rows_per_sample", 0), rowvec_ld=a.get("rowvec_ld", 0), residual=res,
                     geglu=geglu, bn=a.get("bn", 0), gn_stats=st.view.view(-1, n, 2) if st else None,
                     **{key: o.arg for key, o in outs.items()}, **kw)
        be.sync()
        for key, o in outs.items():
            o.check(key)
            _finite(key, o.view)
        if st is not None:
            st.check("gn_stats")
        got = {key: o.view for key, o in outs.items()}
        return got, (a0, rowvec, res, st.view.view(-1, n, 2) if st else None)

    b_all = list(range(b))
    got, (a0, rowvec, res, st) = launch(b_all, "main")
    sel = _sel(b)
    x = _rows(a0, sel, per_in).double()
    wr = w.to(BF16).double().to(be.dev)
    y = _conv_ref(x.reshape(len(sel), conv[1] * stride, conv[2] * stride, c0), wr, stride, taps) if conv else x @ wr
    if bias is not None:
        y += bias.double().to(be.dev)
    if rowvec is not None:
        y += torch.repeat_interleave(rowvec[sel].double(), per_out, 0)
    if res is not None:
        y += _rows(res, sel, per_out).double()
    if geglu:
        lin, gate = y[:, :n // 2], y[:, n // 2:]
        check_close("out_bf16", _rows(got["out_bf16"], sel, per_out), lin * _gelu_tanh(gate), BF16_MAX, BF16_L2)
        if "aux_bf16" in got:
            t = _rows(got["aux_bf16"], sel, per_out).reshape(-1, n // a["bn"], 2, a["bn"] // 2)
            plain = torch.cat([t[:, :, 0].reshape(-1, n // 2), t[:, :, 1].reshape(-1, n // 2)], 1)
            check_close("aux_bf16", plain, y, BF16_MAX, BF16_L2)
    else:
        if "out_f32" in got:
            check_close("out_f32", _rows(got["out_f32"], sel, per_out), y, F32_MAX, F32_L2)
        if "out_bf16" in got:
            check_close("out_bf16", _rows(got["out_bf16"], sel, per_out), y, BF16_MAX, BF16_L2)
            if "out_f32" in got:
                assert torch.equal(got["out_bf16"], got["out_f32"].to(BF16)), "out_bf16 is not out_f32 rounded"
    if st is not None:
        _slab_check("gn_stats", st, got["out_f32"])
    _bit_checks(be, b, lambda seeds, variant: launch(seeds, variant)[0], per_out)


# ------------------------------------------------------------------------------------------------- norms ------
def _designed(be, seeds, rows, c, salt):
    """the residual stream's distribution: per (sample, channel) offset and scale"""
    out = []
    for s in seeds:
        g = torch.Generator(device=be.dev).manual_seed(1_000_003 * salt + s)
        shift = torch.randn(c, generator=g, device=be.dev) * 2.0
        scale = torch.exp(0.5 * torch.randn(c, generator=g, device=be.dev))
        out.append(torch.randn(rows, c, generator=g, device=be.dev) * scale + shift)
    return torch.cat(out)


def _produce(be, seeds, hw, c, salt, with_stats):
    """fp32 [B*hw, c] stream tensor written by a linear igemm (K = 64) whose residual carries the designed
    distribution, with the slab statistics its epilogue leaves for the GroupNorm"""
    m = len(seeds) * hw
    g = torch.Generator().manual_seed(salt)
    wt = (torch.randn(c, 64, generator=g) * 0.05).to(BF16).to(be.dev)
    a0 = _seeded(be, seeds, hw, 64, salt + 7).to(BF16)
    x = torch.empty(m, c, device=be.dev)
    st = torch.empty(census_mod.real_ops.gn_stats_shape(m, c), device=be.dev) if with_stats else None
    be.ops.igemm(a0=a0, wt=wt, n=c, c0=64, m=m, residual=_designed(be, seeds, hw, c, salt), out_f32=x, gn_stats=st)
    be.sync()
    return x, st


def _gn_ref(x, sc, bi, s, hw, silu):
    c = x.shape[1]
    y = F.group_norm(x.double().reshape(s, hw, c).permute(0, 2, 1), 32, sc.double(), bi.double(), 1e-5)
    y = y.permute(0, 2, 1).reshape(-1, c)
    return F.silu(y) if silu else y


def _gn_launch(be, x0, x1, st0, st1, sc, bi, bb, hw, c0, c1, silu, outs_wanted):
    m, c = bb * hw, c0 + c1
    ws = torch.zeros(be.ops.groupnorm_workspace_floats(bb, hw, c), device=be.dev)
    outs = {k: Guarded(m, c, F32 if k == "y_f32" else BF16, be.dev) for k in outs_wanted}
    be.ops.groupnorm_fwd(x0, sc, bi, ws, bb, hw, c0, x1=x1, c1=c1, silu=silu, stats0=st0, stats1=st1,
                         **{k: o.view for k, o in outs.items()})
    be.sync()
    for k, o in outs.items():
        o.check(k)
        _finite(k, o.view)
    return {k: o.view for k, o in outs.items()}


def replay_groupnorm_fwd(be, call):
    a, b = call.args, call.batch
    hw, c0, c1, silu = a["hw"], a["c0"], a.get("c1", 0), a.get("silu", True)
    c = c0 + c1
    stats = a.get("stats0") is not None
    assert (a.get("stats1") is not None) == (stats and c1 > 0)
    wanted = [k for k in ("y_bf16", "y_f32", "raw_bf16") if a.get(k) is not None]
    g = torch.Generator().manual_seed(hw + c)
    sc = (1.0 + 0.1 * torch.randn(c, generator=g)).to(be.dev)
    bi = (0.1 * torch.randn(c, generator=g)).to(be.dev)

    def make(seeds, with_stats):
        x0, st0 = _produce(be, seeds, hw, c0, 11, with_stats)
        x1, st1 = _produce(be, seeds, hw, c1, 13, with_stats) if c1 else (None, None)
        return x0, x1, st0, st1

    def launch(seeds):
        x0, x1, st0, st1 = make(seeds, stats)
        return _gn_launch(be, x0, x1, st0, st1, sc, bi, len(seeds), hw, c0, c1, silu, wanted)

    x0, x1, st0, st1 = make(list(range(b)), stats)
    got = _gn_launch(be, x0, x1, st0, st1, sc, bi, b, hw, c0, c1, silu, wanted)
    two_pass = _gn_launch(be, x0, x1, None, None, sc, bi, b, hw, c0, c1, silu, wanted)
    sel = _sel(b)
    x = x0 if x1 is None else torch.cat([x0, x1], 1)
    ref = _gn_ref(_rows(x, sel, hw), sc, bi, len(sel), hw, silu)
    for name, outs in (("", got), ("two-pass ", two_pass)):
        if "y_bf16" in outs:
            check_close(name + "y_bf16", _rows(outs["y_bf16"], sel, hw), ref, BF16_MAX, BF16_L2)
        if "y_f32" in outs:
            check_close(name + "y_f32", _rows(outs["y_f32"], sel, hw), ref, F32_MAX, F32_L2)
        if "raw_bf16" in outs:
            assert torch.equal(outs["raw_bf16"], x.to(BF16)), "raw_bf16 is not the input rounded to bf16"
    if be.emulated:
        return
    for k in got:
        _same_bits(f"{k} rerun", launch(list(range(b)))[k], got[k])
    for s in (0, b - 1):        # sample s alone on its own rows of the batch's input and statistics
        rows = slice(s * hw, (s + 1) * hw)
        slabs = slice(s * hw // 32, (s + 1) * hw // 32)
        alone = _gn_launch(be, x0[rows].contiguous(), x1[rows].contiguous() if c1 else None,
                           st0[slabs].contiguous() if stats else None, st1[slabs].contiguous() if st1 is not None else None,
                           sc, bi, 1, hw, c0, c1, silu, wanted)
        for k in alone:
            _same_bits(f"{k} of sample {s} alone", alone[k], got[k][rows])
    if b in OTHER_BATCH:
        other = launch(_other_seeds(b))
        for k in other:
            for i, s in enumerate((b - 1, 0)):
                _same_bits(f"{k} of sample {s} at batch {OTHER_BATCH[b]}", other[k][i * hw:(i + 1) * hw],
                           got[k][s * hw:(s + 1) * hw])


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


# ----------------------------------------------------------------------------------------- exact ops ------
def replay_cast_bf16(be, call):
    a, b = call.args, call.batch
    shape = a["x"].shape
    cols = shape[-1]
    rows = math.prod(shape) // cols
    x = _seeded(be, list(range(b)), rows // b, cols, 29, scale=3.0)
    # exact ties between two bf16 neighbours (round to the even one) and values at the ends of the bf16 range
    base = x[:1].to(BF16).float()
    x[:1] = (base + (base.view(torch.int32) + 65536).view(F32)) / 2
    x[1, :4] = torch.tensor([3.3e38, -3.3e38, 1e-40, -0.0])
    y = Guarded(rows, cols, BF16, be.dev)
    be.ops.cast_bf16(x.view(-1, *shape[1:]), y.view)
    be.sync()
    y.check("y")
    _same_bits("cast_bf16 against round-to-nearest-even", y.view, x.to(BF16))


def replay_upsample2x_bf16(be, call):
    a, b = call.args, call.batch
    h, w, c = a["h"], a["w"], a["c"]
    x = _seeded(be, list(range(b)), h * w, c, 31, scale=3.0)
    y = Guarded(b * 4 * h * w, c, BF16, be.dev)
    be.ops.upsample2x_bf16(x, y.view, b, h, w, c)
    be.sync()
    y.check("y")
    ref = x.reshape(b, h, w, c).repeat_interleave(2, 1).repeat_interleave(2, 2).reshape(-1, c).to(BF16)
    _same_bits("upsample2x_bf16 against the bf16 nearest-neighbour repeat", y.view, ref)


# ---------------------------------------------------------------------------------------------- sums ------
def replay_conv_in(be, call):
    a, b = call.args, call.batch
    cin, h, wd, cout = a["cin"], a["h"], a["wd"], a["cout"]
    g = torch.Generator().manual_seed(37)
    w = (torch.randn(3, 3, cin, cout, generator=g) * (9 * cin) ** -0.5).to(be.dev)
    bias = (torch.randn(cout, generator=g) * 0.5).to(be.dev)

    def launch(seeds, variant):
        bb = len(seeds)
        lat = _seeded(be, seeds, cin, h * wd, 41, scale=1.5).reshape(bb, cin, h, wd)
        y = Guarded(bb * h * wd, cout, F32, be.dev)
        st = Guarded(-(-bb * h * wd // 32), 2 * cout, F32, be.dev) \
            if a.get("gn_stats") is not None and variant == "main" else None
        be.ops.conv_in(lat, w, bias, y.view, bb, cin, h, wd, cout, gn_stats=st.view.view(-1, cout, 2) if st else None)
        be.sync()
        y.check("y")
        _finite("y", y.view)
        if st:
            st.check("gn_stats")
        return {"y": y.view}, lat, (st.view.view(-1, cout, 2) if st else None)

    got, lat, st = launch(list(range(b)), "main")
    sel = _sel(b)
    x = lat[sel].double().permute(0, 2, 3, 1)
    wr = w.double().reshape(9 * cin, cout)
    ref = _conv_ref(x, wr, 1, 9) + bias.double()
    terms = _conv_ref(x.abs(), wr.abs(), 1, 9) + bias.double().abs()
    check_sum("y", _rows(got["y"], sel, h * wd), ref, terms)
    if st is not None:
        _slab_check("gn_stats", st, got["y"])
    _bit_checks(be, b, lambda seeds, variant: launch(seeds, variant)[0], h * wd)


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
def _torch_f32_error(x, fn_ref, fn32):
    """max and L2 error, relative to the float64 result, of the same normalisation computed in torch fp32 with
    var = mean(x^2) - mean(x)^2: what the statistics' formulation itself costs at this input"""
    ref, y32 = fn_ref(x), fn32(x)
    d = y32.double() - ref
    return (d.abs().max() / ref.abs().max()).item(), (d.norm() / ref.norm()).item()


def _check_vs_f32(name, out, ref, e32, max_tol, l2_tol):
    d = out.double() - ref
    e_max, e_l2 = (d.abs().max() / ref.abs().max()).item(), (d.norm() / ref.norm()).item()
    bmax, bl2 = max(max_tol, NORM_DC_FACTOR * e32[0]), max(l2_tol, NORM_DC_FACTOR * e32[1])
    _record(name, max=e_max, l2=e_l2, torch_f32_max=e32[0], torch_f32_l2=e32[1])
    assert e_max <= bmax and e_l2 <= bl2, f"{name}: max err {e_max:.3g} (bound {bmax:.3g}), L2 {e_l2:.3g} (bound {bl2:.3g})"


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


def _produce_unit(be, seeds, hw, c, dc):
    """like _produce, with a unit-variance residual (per-channel scale 1, no per-channel shift) plus the offset dc"""
    m = len(seeds) * hw
    wt = torch.zeros(c, 64, dtype=BF16, device=be.dev)
    a0 = torch.zeros(m, 64, dtype=BF16, device=be.dev)
    x = torch.empty(m, c, device=be.dev)
    st = torch.empty(census_mod.real_ops.gn_stats_shape(m, c), device=be.dev)
    be.ops.igemm(a0=a0, wt=wt, n=c, c0=64, m=m, residual=_seeded(be, seeds, hw, c, 71) + dc, out_f32=x, gn_stats=st)
    be.sync()
    return x, st


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
