"""Replays of forward launches that the U-Net and the VAE share (igemm, GroupNorm, conv_in, cast_bf16,
upsample2x_bf16), and the helpers they need: test_forward_layers.py and test_vae_layers.py replay the configurations
tests/_forward_census.py records with these.  Each replay runs one recorded launch on a backend (the CUDA library or its
torch-CPU emulation) and checks it against a float64 reference fed the same bf16-rounded operands; on the CUDA library
it also checks bits across reruns, a sample alone against its rows of the batch, and a sample at the model's other
batch size (``other_batch``: {16: 40, 40: 16} for the U-Net's sampling and train passes, {2: 1, 1: 2} for a VAE chunk
of 2 and the tail chunk of 1)."""
import math

import torch
import torch.nn.functional as F
import _forward_census as census_mod
from _layer_check import (BF16, BF16_L2, BF16_MAX, F32, F32_L2, F32_MAX, NORM_DC_FACTOR, Guarded, _record, check_close,
                          check_sum)

OTHER_BATCH = {16: 40, 40: 16}      # the U-Net's two batch sizes: sampling (2 x 8 for CFG) and the PPO train pass


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
    return sorted(s for s in {0, 1, b // 2, b - 1} if s < b)


def _ends(b):
    """the samples the bit checks follow: B-1 and 0"""
    return list(dict.fromkeys((b - 1, 0)))


def _other_seeds(b, b2):
    """seeds of a launch at batch b2: the first of ``_ends(b)`` that fit, fresh seeds after them"""
    first = _ends(b)[:b2]
    return first + [10_000 + i for i in range(b2 - len(first))]


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


def _bit_checks(be, b, launch, per, other_batch=OTHER_BATCH):
    """launch(seeds, variant) -> {name: [rows, ...] tensor, ``per`` rows per sample}; variant "main" as recorded, "rerun"
    without optional side outputs that must not change the main ones, "other" (at batch ``other_batch[b]``) with the
    train pass's extra outputs toggled"""
    if be.emulated:
        return
    ref = launch(list(range(b)), "main")
    again = launch(list(range(b)), "rerun")
    for k in again:
        _same_bits(f"{k} rerun", again[k], ref[k])
    for s in sorted(_ends(b)):
        alone = launch([s], "rerun")
        for k in alone:
            _same_bits(f"{k} of sample {s} alone", alone[k], ref[k][s * per:(s + 1) * per])
    if b in other_batch:
        b2 = other_batch[b]
        other = launch(_other_seeds(b, b2), "other")
        for k in other:
            for i, s in enumerate(_ends(b)[:b2]):
                if k in ref:
                    _same_bits(f"{k} of sample {s} at batch {b2}", other[k][i * per:(i + 1) * per],
                               ref[k][s * per:(s + 1) * per])


def _conv_ref(x, w, stride, taps, no_low_pad=False):
    """float64 conv of NHWC x [S, Hi, Wi, Cin] with the natural kernel w [taps * Cin, N] ((ky, kx, cin) rows), padding 1
    for 3x3 (with ``no_low_pad``, as the VAE encoder's down-sample: padding (0, 1), on the high side only): one float64
    GEMM per tap"""
    s, hi, wi, cin = x.shape
    n = w.shape[1]
    if taps == 1:
        return x.reshape(-1, cin) @ w
    ho, wo = hi // stride, wi // stride
    xp = F.pad(x, (0, 0, 0, 1, 0, 1) if no_low_pad else (0, 0, 1, 1, 1, 1))
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


def replay_igemm(be, call, other_batch=OTHER_BATCH):
    a, b = call.args, call.batch
    assert call.role is None, "the VAE attention's GEMMs have replays of their own (test_vae_layers.py)"
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
                     no_low_pad=bool(a.get("no_low_pad")), **{key: o.arg for key, o in outs.items()}, **kw)
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
    y = _conv_ref(x.reshape(len(sel), conv[1] * stride, conv[2] * stride, c0), wr, stride, taps,
                  bool(a.get("no_low_pad"))) if conv else x @ wr
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
    _bit_checks(be, b, lambda seeds, variant: launch(seeds, variant)[0], per_out, other_batch)


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


def _gn_ref(x, sc, bi, s, hw, silu, eps=1e-5):
    c = x.shape[1]
    y = F.group_norm(x.double().reshape(s, hw, c).permute(0, 2, 1), 32, sc.double(), bi.double(), eps)
    y = y.permute(0, 2, 1).reshape(-1, c)
    return F.silu(y) if silu else y


def _gn_launch(be, x0, x1, st0, st1, sc, bi, bb, hw, c0, c1, silu, outs_wanted, eps=1e-5):
    m, c = bb * hw, c0 + c1
    ws = torch.zeros(be.ops.groupnorm_workspace_floats(bb, hw, c), device=be.dev)
    outs = {k: Guarded(m, c, F32 if k == "y_f32" else BF16, be.dev) for k in outs_wanted}
    be.ops.groupnorm_fwd(x0, sc, bi, ws, bb, hw, c0, x1=x1, c1=c1, silu=silu, stats0=st0, stats1=st1, eps=eps,
                         **{k: o.view for k, o in outs.items()})
    be.sync()
    for k, o in outs.items():
        o.check(k)
        _finite(k, o.view)
    return {k: o.view for k, o in outs.items()}


def replay_groupnorm_fwd(be, call, other_batch=OTHER_BATCH):
    a, b = call.args, call.batch
    hw, c0, c1, silu, eps = a["hw"], a["c0"], a.get("c1", 0), a.get("silu", True), a.get("eps", 1e-5)
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
        return _gn_launch(be, x0, x1, st0, st1, sc, bi, len(seeds), hw, c0, c1, silu, wanted, eps)

    x0, x1, st0, st1 = make(list(range(b)), stats)
    got = _gn_launch(be, x0, x1, st0, st1, sc, bi, b, hw, c0, c1, silu, wanted, eps)
    two_pass = _gn_launch(be, x0, x1, None, None, sc, bi, b, hw, c0, c1, silu, wanted, eps)
    sel = _sel(b)
    x = x0 if x1 is None else torch.cat([x0, x1], 1)
    ref = _gn_ref(_rows(x, sel, hw), sc, bi, len(sel), hw, silu, eps)
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
    for s in sorted(_ends(b)):        # sample s alone on its own rows of the batch's input and statistics
        rows = slice(s * hw, (s + 1) * hw)
        slabs = slice(s * hw // 32, (s + 1) * hw // 32)
        alone = _gn_launch(be, x0[rows].contiguous(), x1[rows].contiguous() if c1 else None,
                           st0[slabs].contiguous() if stats else None, st1[slabs].contiguous() if st1 is not None else None,
                           sc, bi, 1, hw, c0, c1, silu, wanted, eps)
        for k in alone:
            _same_bits(f"{k} of sample {s} alone", alone[k], got[k][rows])
    if b in other_batch:
        b2 = other_batch[b]
        other = launch(_other_seeds(b, b2))
        for k in other:
            for i, s in enumerate(_ends(b)[:b2]):
                _same_bits(f"{k} of sample {s} at batch {b2}", other[k][i * hw:(i + 1) * hw],
                           got[k][s * hw:(s + 1) * hw])


# ----------------------------------------------------------------------------------------- exact ops ------
def replay_cast_bf16(be, call, other_batch=OTHER_BATCH):
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


def replay_upsample2x_bf16(be, call, other_batch=OTHER_BATCH):
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
def replay_conv_in(be, call, other_batch=OTHER_BATCH):
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
    _bit_checks(be, b, lambda seeds, variant: launch(seeds, variant)[0], h * wd, other_batch)


def _produce_unit(be, seeds, hw, c, dc, sigma=1.0):
    """like _produce, with a residual of standard deviation ``sigma`` (the same in every channel, no per-channel shift)
    plus the offset dc"""
    m = len(seeds) * hw
    wt = torch.zeros(c, 64, dtype=BF16, device=be.dev)
    a0 = torch.zeros(m, 64, dtype=BF16, device=be.dev)
    x = torch.empty(m, c, device=be.dev)
    st = torch.empty(census_mod.real_ops.gn_stats_shape(m, c), device=be.dev)
    be.ops.igemm(a0=a0, wt=wt, n=c, c0=64, m=m, residual=_seeded(be, seeds, hw, c, 71, scale=sigma) + dc, out_f32=x,
                 gn_stats=st)
    be.sync()
    return x, st


# ----------------------------------------------------------------- norms fed inputs whose statistics cancel ------
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
