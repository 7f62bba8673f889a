"""The VAE (ddpo_b200/vae.py, ``VAEDecoder.decode`` and ``VAEEncoder.encode``) launch by launch: every distinct kernel
configuration the SD VAE launches at 512 px, at the production chunk of 2 images and at the tail chunk of 1, replayed on
the CUDA library against a float64 reference fed the same bf16-rounded operands.  The configurations come from
tests/_forward_census.py (``vae_census``), which records the decoder's and encoder's launches on the ``meta`` device.
The ops the U-Net launches too replay with tests/_forward_replays.py; the VAE-only ops (the mid-block attention's score
GEMMs and row softmax, post_quant, conv_out with the image post-processing, the encoder's input transpose and head) have
replays here.  The VAE_MICRO configurations replay on the torch-CPU emulation of the ops (value checks only) in the CPU
suite.

Every replay keeps the bit-level checks of the U-Net census: a rerun gives the same bits, samples 0 and B-1 computed
alone equal their rows of the batch, and a sample gives the same bits at chunk batch 1 and 2.  The attention's score
GEMMs and softmax run once per sample whatever the chunk batch; their replays check that a sample's rows taken from a
two-sample buffer give the same bits as the sample alone.

Also here: GroupNorm at the VAE's statistics sizes (1 M elements per group at 512 px, eps 1e-6), and the whole decoder
and encoder at 512 px against the float64 oracle on the GPU, with the uint8 images the rewards consume."""
import collections

import numpy as np
import pytest
import torch
import torch.nn.functional as F
import _forward_census as census_mod
from _forward_replays import (_bit_checks, _check_vs_f32, _conv_ref, _designed, _finite, _gn_launch, _gn_ref,
                              _produce_unit, _rows, _same_bits, _seeded, _sel, _torch_f32_error, replay_cast_bf16,
                              replay_conv_in, replay_groupnorm_fwd, replay_igemm, replay_upsample2x_bf16)
from _layer_check import (BF16, BF16_L2, BF16_MAX, F32, F32_L2, F32_MAX, Backend, Guarded, _current_node,  # noqa: F401
                          _record, check_close, check_sum)
from ddpo_b200 import vae as vae_mod

VAE_OTHER_BATCH = {2: 1, 1: 2}      # the decoder's chunk of 2 (decode_batch) and the tail chunk of an odd batch
BF16_REL = 2.0 ** -8 + 1e-5         # one bf16 rounding (half an ulp <= 2^-8 of the value) plus fp32 arithmetic


def _uniform(be, seeds, rows, cols, salt):
    """[len(seeds) * rows, cols] uniform in [0, 1), per sample from its seed"""
    out = []
    for s in seeds:
        g = torch.Generator(device=be.dev).manual_seed(1_000_003 * salt + s)
        out.append(torch.rand(rows, cols, generator=g, device=be.dev))
    return torch.cat(out)


class _RowSlot:
    """rows [s * per, (s + 1) * per) of a [b * per, cols] buffer (plus 8 rows after it) of seeded noise, the way
    ``_attention`` hands one sample's rows of ``ao`` to the P V GEMM; everything outside the slot must come back
    unchanged"""

    def __init__(self, b, s, per, cols, dtype, dev):
        self.g = Guarded(b * per, cols, dtype, dev)
        self.rows = slice(s * per, (s + 1) * per)

    @property
    def view(self):
        return self.g.buf[self.rows]

    def check(self, what):
        outside = torch.ones(self.g.buf.shape[0], dtype=torch.bool, device=self.g.buf.device)
        outside[self.rows] = False
        assert torch.equal(self.g.buf[outside], self.g.snapshot[outside]), f"{what}: write outside the sample's rows"


# ------------------------------------------------------------------------------------- the attention block ------
def replay_attention_gemm(be, call, other_batch=VAE_OTHER_BATCH):
    """One of the three GEMMs of ``_attention``'s per-sample loop, with its operands as that loop builds them:
    "vt": V^T [c, hw] with the prepared value weight as the row operand and the sample's GroupNorm'd rows as ``wt``;
    "qk": Q K^T [hw, hw] fp32 from the sample's q and k rows; "pv": P V + value bias into the sample's rows of ``ao``,
    with P a softmax output (non-negative rows that sum to 1) and V^T as ``wt``."""
    a, role = call.args, call.role
    assert call.batch == 1 and a.get("conv") is None and a.get("residual") is None
    m, n, c0 = a["m"], a["n"], a["c0"]
    hw, c = {"vt": (n, m), "qk": (m, c0), "pv": (m, n)}[role]
    g = torch.Generator().manual_seed(hw + 7 * c)
    wv = torch.randn(c, c, generator=g) * c ** -0.5               # natural layout [c_in, c_out]
    bias = torch.randn(c, generator=g) * 0.5 if a.get("bias") is not None else None
    wv_t = torch.empty(c, c, dtype=BF16, device=be.dev)
    be.ops.prep_weight(wv.to(be.dev), wv_t, c, c)

    def sample(seed, salt, rows, cols):
        return _seeded(be, [seed], rows, cols, salt).to(BF16)

    def probs(seed):
        q, k = sample(seed, 113, hw, c), sample(seed, 127, hw, c)
        return torch.softmax(q.float() @ k.float().t() * c ** -0.5, -1).to(BF16)

    def slots(make, s, nb):
        """the operand of sample ``seed`` 0 at slot s of an nb-sample buffer (other slots: other seeds)"""
        return torch.cat([make(0 if i == s else 500 + i) for i in range(nb)])

    def launch(s, nb):
        """sample (seed 0) at slot s of a chunk of nb: its per-sample operand rows are rows s of nb-sample buffers"""
        if role == "vt":
            gb = slots(lambda sd: sample(sd, 109, hw, c), s, nb)
            args, ops_in = dict(a0=wv_t, wt=gb[s * hw:(s + 1) * hw]), (gb[s * hw:(s + 1) * hw],)
            out = Guarded(c, hw, BF16, be.dev)
        elif role == "qk":
            qb = slots(lambda sd: sample(sd, 113, hw, c), s, nb)
            kb = slots(lambda sd: sample(sd, 127, hw, c), s, nb)
            rows = slice(s * hw, (s + 1) * hw)
            args, ops_in = dict(a0=qb[rows], wt=kb[rows]), (qb[rows], kb[rows])
            out = Guarded(hw, hw, F32, be.dev)
        else:
            p, vt = probs(0), sample(0, 131, c, hw)
            args, ops_in = dict(a0=p, wt=vt, bias=bias.to(be.dev)), (p, vt)
            out = _RowSlot(nb, s, hw, c, BF16, be.dev)
        key = "out_f32" if role == "qk" else "out_bf16"
        be.ops.igemm(n=n, c0=c0, m=m, **args, **{key: out.view})
        be.sync()
        out.check(key)
        _finite(key, out.view)
        return out.view, ops_in

    got, ops_in = launch(0, 1)
    if role == "vt":
        ref = (ops_in[0].double() @ wv.to(BF16).double().to(be.dev)).t()
        check_close("vt out_bf16", got, ref, BF16_MAX, BF16_L2)
    elif role == "qk":
        check_close("qk out_f32", got, ops_in[0].double() @ ops_in[1].double().t(), F32_MAX, F32_L2)
    else:
        p, vt = ops_in
        assert (p.float() >= 0).all() and ((p.double().sum(-1) - 1).abs() <= BF16_REL).all()
        ref = p.double() @ vt.double().t() + bias.double().to(be.dev)
        check_close("pv out_bf16", got, ref, BF16_MAX, BF16_L2)
    if be.emulated:
        return
    _same_bits(f"{role} rerun", launch(0, 1)[0], got)
    for s in range(2):
        _same_bits(f"{role} of a sample at slot {s} of a chunk of 2", launch(s, 2)[0], got)


def replay_softmax_rows(be, call, other_batch=VAE_OTHER_BATCH):
    """P = softmax(scale * S) per row, bf16, for the scores the block produces (q, k of a GroupNorm'd input: logits
    ~ N(0, 1) at scale c^-1/2) and for rows where one entry takes almost all the mass (one logit raised by 30)"""
    a = call.args
    rows, n = a["scores"].shape
    scale = a["scale"]
    c = round(scale ** -2)
    assert call.batch == 1 and abs(c ** -0.5 - scale) < 1e-6 * scale

    def scores(peaked):
        q = _seeded(be, [0], rows, c, 137).to(BF16).float()
        k = _seeded(be, [0], n, c, 139).to(BF16).float()
        s = q @ k.t()
        if peaked:
            r = torch.arange(rows, device=be.dev)
            s[r, (r * 7919) % n] += 30.0 / scale
        return s

    def launch(s):
        p = Guarded(s.shape[0], n, BF16, be.dev)
        be.ops.softmax_rows(s, p.view, scale)
        be.sync()
        p.check("probs")
        _finite("probs", p.view)
        return p.view

    for kind in ("block", "peaked"):
        s = scores(kind == "peaked")
        got = launch(s)
        ref = torch.softmax(s.double() * scale, -1)
        check_close(f"{kind} probs", got, ref, BF16_MAX, BF16_L2)
        rel = ((got.double() - ref).abs() / (BF16_REL * ref)).max().item()
        _record(f"{kind} probs elementwise", worst_over_bound=rel)
        assert rel <= 1.0, f"{kind}: elementwise error {rel:.3g} x (2^-8 of the value)"
        sums = (got.double().sum(-1) - 1).abs().max().item()
        _record(f"{kind} row sums", worst_over_bound=sums / BF16_REL)
        assert sums <= BF16_REL, f"{kind}: a row sums to 1 +- {sums:.3g}"
        if kind == "peaked":
            assert (ref.max(-1).values > 0.999).all()
        if be.emulated:
            continue
        _same_bits(f"{kind} rerun", launch(s), got)
        for r in (0, rows - 1):         # one CTA per row: a row alone gives its bits in the full launch
            _same_bits(f"{kind} row {r} alone", launch(s[r:r + 1].contiguous()), got[r:r + 1])


# ------------------------------------------------------------------------------------- the VAE-only ops ------
def replay_vae_post_quant(be, call, other_batch=VAE_OTHER_BATCH):
    """z = post_quant_conv(latents / 0.18215): the 1x1 4 -> 4 conv on NCHW latents"""
    a, b = call.args, call.batch
    _, lc, h, wd = a["latents"].shape
    scaling = a.get("scaling", vae_mod.VAE_SCALING)
    g = torch.Generator().manual_seed(149)
    w = torch.randn(1, 1, lc, lc, generator=g).to(be.dev)
    bias = (torch.randn(lc, generator=g) * 0.5).to(be.dev)

    def launch(seeds, variant):
        bb = len(seeds)
        lat = _seeded(be, seeds, lc, h * wd, 151, scale=scaling).reshape(bb, lc, h, wd)
        out = Guarded(bb * lc, h * wd, F32, be.dev)
        be.ops.vae_post_quant(lat, w, bias, out.view.view(bb, lc, h, wd), scaling=scaling)
        be.sync()
        out.check("z")
        _finite("z", out.view)
        return {"z": out.view}, lat

    got, lat = launch(list(range(b)), "main")
    z = lat.double() / scaling
    wd64 = w.double().reshape(lc, lc)
    ref = torch.einsum("bihw,io->bohw", z, wd64) + bias.double()[None, :, None, None]
    terms = torch.einsum("bihw,io->bohw", z.abs(), wd64.abs()) + bias.double().abs()[None, :, None, None]
    check_sum("z", got["z"], ref.reshape(-1, h * wd), terms.reshape(-1, h * wd))
    _bit_checks(be, b, lambda seeds, variant: launch(seeds, variant)[0], lc, other_batch)


def replay_vae_conv_out(be, call, other_batch=VAE_OTHER_BATCH):
    """the decoder's conv_out (3x3, c -> 3) with the image post-processing: ``raw_nchw`` (the decoder's .sample) against
    float64, ``img_nhwc`` as clip(raw / 2 + 0.5, 0, 1) with raw past both clip ends; each output also alone"""
    a, b = call.args, call.batch
    h, wd, cin = a["h"], a["wd"], a["cin"]
    g = torch.Generator().manual_seed(157)
    w = (torch.randn(3, 3, cin, 3, generator=g) * (9 * cin) ** -0.5).to(be.dev)
    bias = torch.tensor([0.3, -0.2, 0.1]).to(be.dev)

    def launch(seeds, variant, outs=("raw", "img")):
        bb = len(seeds)
        x = F.silu(_designed(be, seeds, h * wd, cin, 163))
        raw = Guarded(bb * 3 * h, wd, F32, be.dev) if "raw" in outs else None
        img = Guarded(bb * h * wd, 3, F32, be.dev) if "img" in outs else None
        be.ops.vae_conv_out(x, w, bias, bb, h, wd, cin, raw_nchw=raw.view.view(bb, 3, h, wd) if raw else None,
                            img_nhwc=img.view.view(bb, h, wd, 3) if img else None)
        be.sync()
        res = {}
        for k, o in (("raw", raw), ("img", img)):
            if o is not None:
                o.check(k)
                _finite(k, o.view)
                res[k] = o.view.reshape(bb, -1)
        return res, x

    got, x = launch(list(range(b)), "main")
    sel = _sel(b)
    xs = _rows(x, sel, h * wd).double().reshape(len(sel), h, wd, cin)
    wr = w.double().reshape(9 * cin, 3)
    nchw = lambda t: t.reshape(len(sel), h, wd, 3).permute(0, 3, 1, 2).reshape(len(sel), -1)
    ref = _conv_ref(xs, wr, 1, 9) + bias.double()
    terms = _conv_ref(xs.abs(), wr.abs(), 1, 9) + bias.double().abs()
    assert (ref < -1).any() and (ref > 1).any(), "raw does not reach past both clip ends"
    check_sum("raw_nchw", got["raw"][sel], nchw(ref), nchw(terms))
    # |clip(r / 2 + 0.5) - clip(ref / 2 + 0.5)| <= |r - ref| / 2, plus the rounding of the + 0.5
    ref_img = (ref / 2 + 0.5).clamp(0, 1).reshape(len(sel), -1)
    check_sum("img_nhwc", got["img"][sel], ref_img, (terms / 2 + 0.5).reshape(len(sel), -1))
    _same_bits("img_nhwc against clip(raw * 0.5 + 0.5, 0, 1)", got["img"],
               (got["raw"].reshape(b, 3, h, wd).permute(0, 2, 3, 1) * 0.5 + 0.5).clamp(0, 1).reshape(b, -1))
    assert (got["img"] == 0).any() and (got["img"] == 1).any()
    for only in ("raw", "img"):
        _same_bits(f"{only} without the other output", launch(list(range(b)), "main", (only,))[0][only], got[only])
    _bit_checks(be, b, lambda seeds, variant: launch(seeds, variant)[0], 1, other_batch)


def replay_vae_image_to_nchw(be, call, other_batch=VAE_OTHER_BATCH):
    """(images - 0.5) / 0.5, NHWC -> NCHW: bit-exact against the same fp32 arithmetic"""
    a, b = call.args, call.batch
    _, h, wd, _ = a["img_nhwc"].shape

    def launch(seeds, variant):
        bb = len(seeds)
        img = _uniform(be, seeds, h * wd, 3, 167)
        edges = torch.tensor([0.0, 1.0, 0.5, float(np.nextafter(np.float32(0.5), np.float32(0)))], device=be.dev)
        img.view(bb, h * wd, 3)[:, :4, 0] = edges         # in every sample, so that its bits do not depend on its slot
        out = Guarded(bb * 3 * h, wd, F32, be.dev)
        be.ops.vae_image_to_nchw(img.view(bb, h, wd, 3), out.view.view(bb, 3, h, wd))
        be.sync()
        out.check("out")
        _same_bits("image_to_nchw against (x - 0.5) / 0.5", out.view,
                   ((img - 0.5) / 0.5).view(bb, h, wd, 3).permute(0, 3, 1, 2).reshape(-1, wd))
        return {"out": out.view}

    launch(list(range(b)), "main")
    _bit_checks(be, b, launch, 3 * h, other_batch)


def replay_vae_encoder_head(be, call, other_batch=VAE_OTHER_BATCH):
    """the encoder's fp32 head: 3x3 conv c -> 8, quant_conv 1x1 8 -> 8, logvar half clipped to [-30, 20], with both
    clip bounds reached"""
    a, b = call.args, call.batch
    h, wd, cin = a["h"], a["wd"], a["cin"]
    g = torch.Generator().manual_seed(173)
    w = (torch.randn(3, 3, cin, 8, generator=g) * (9 * cin) ** -0.5).to(be.dev)
    bias = (torch.randn(8, generator=g) * 0.5).to(be.dev)
    wq = (torch.randn(1, 1, 8, 8, generator=g) * 20).to(be.dev)
    bq = torch.randn(8, generator=g).to(be.dev)

    def launch(seeds, variant):
        bb = len(seeds)
        x = F.silu(_designed(be, seeds, h * wd, cin, 179))
        mom = Guarded(bb * h * wd, 8, F32, be.dev)
        be.ops.vae_encoder_head(x, w, bias, wq, bq, mom.view.view(bb, h, wd, 8), bb, h, wd, cin)
        be.sync()
        mom.check("moments")
        _finite("moments", mom.view)
        return {"moments": mom.view}, x

    got, x = launch(list(range(b)), "main")
    sel = _sel(b)
    xs = _rows(x, sel, h * wd).double().reshape(len(sel), h, wd, cin)
    wr, wq64 = w.double().reshape(9 * cin, 8), wq.double().reshape(8, 8)
    hc = _conv_ref(xs, wr, 1, 9) + bias.double()
    m = hc @ wq64 + bq.double()
    ref = torch.cat([m[:, :4], m[:, 4:].clamp(-30.0, 20.0)], 1)
    terms = (_conv_ref(xs.abs(), wr.abs(), 1, 9) + bias.double().abs()) @ wq64.abs() + bq.double().abs()
    assert (m[:, 4:] > 20).any() and (m[:, 4:] < -30).any()
    check_sum("moments", _rows(got["moments"], sel, h * wd), ref, terms)   # the clip is 1-Lipschitz
    logvar = got["moments"][:, 4:]
    assert logvar.max().item() == 20.0 and logvar.min().item() == -30.0
    _bit_checks(be, b, lambda seeds, variant: launch(seeds, variant)[0], h * wd, other_batch)


REPLAY = {"igemm": replay_igemm, "groupnorm_fwd": replay_groupnorm_fwd, "cast_bf16": replay_cast_bf16,
          "upsample2x_bf16": replay_upsample2x_bf16, "conv_in": replay_conv_in, "softmax_rows": replay_softmax_rows,
          "vae_post_quant": replay_vae_post_quant, "vae_conv_out": replay_vae_conv_out,
          "vae_image_to_nchw": replay_vae_image_to_nchw, "vae_encoder_head": replay_vae_encoder_head}
ROLES = ("vt", "qk", "pv")


# ------------------------------------------------------------------------------------------ the census ------
def test_vae_census_starts_and_ends_with_the_models_first_and_last_launches():
    for which in ("full", "micro"):
        for (part, b), calls in census_mod.vae_runs(which).items():
            first, last = ("vae_post_quant", "vae_conv_out") if part == "decoder" else ("vae_image_to_nchw",
                                                                                        "vae_encoder_head")
            assert calls[0].op == first and calls[-1].op == last, (which, part, b)


def test_every_recorded_vae_op_has_a_replay():
    for which in ("full", "micro"):
        calls = [c for _, c, _ in census_mod.vae_census(which)]
        missing = {c.op for c in calls} - set(REPLAY)
        assert not missing, f"VAE ops without a replay in test_vae_layers.py: {sorted(missing)}"
        assert {c.role for c in calls if c.role} == set(ROLES)
        assert all(c.op == "igemm" for c in calls if c.role)


def test_each_vae_signature_has_one_test_id():
    for which in ("full", "micro"):
        entries = census_mod.vae_census(which)
        assert len({k for k, _, _ in entries}) == len(entries)
        ids = [c.test_id() for _, c, _ in entries]
        assert len(set(ids)) == len(ids), which


def test_vae_gemm_launches_match_the_parameter_manifest():
    """per chunk of b images: one implicit GEMM per tensor-core weight (every kernel of the manifest but the CUDA-core
    layers), except the attention's value weight, which the per-sample loop uses as V^T's row operand; per attention
    block and sample a V^T, a Q K^T and a P V GEMM and one row softmax"""
    for which in ("full", "micro"):
        for (part, b), calls in census_mod.vae_runs(which).items():
            cls = vae_mod.VAEDecoder if part == "decoder" else vae_mod.VAEEncoder
            cfg = vae_mod.SD_VAE if which == "full" else vae_mod.VAE_MICRO
            manifest = vae_mod.param_manifest(cfg) if part == "decoder" else vae_mod.encoder_param_manifest(cfg)
            layers = [name[:-len("/kernel")] for name, _ in manifest if name.endswith("/kernel")]
            gemm = [n for n in layers if n not in cls.CUDA_CORE_LAYERS]
            attn = sum(n.endswith("/value") for n in gemm)
            assert attn == 1
            got = collections.Counter(c.role for c in calls if c.op == "igemm")
            assert got == {None: len(gemm) - attn, "vt": b * attn, "qk": b * attn, "pv": b * attn}, (which, part, b)
            assert sum(c.op == "softmax_rows" for c in calls) == b * attn
            assert all(c.batch == (1 if c.role or c.op == "softmax_rows" else b) for c in calls)


def _census_params():
    out = [pytest.param("emulator", c, id="emu-" + c.test_id()) for _, c, _ in census_mod.vae_census("micro")]
    out += [pytest.param("cuda", c, marks=pytest.mark.gpu, id="cuda-" + c.test_id())
            for _, c, _ in census_mod.vae_census("full")]
    return out


@pytest.mark.parametrize("backend,call", _census_params())
def test_vae_launch(backend, call):
    torch.backends.cuda.matmul.allow_tf32 = False
    be = Backend(backend)
    replay = replay_attention_gemm if call.role else REPLAY[call.op]
    replay(be, call, other_batch=VAE_OTHER_BATCH)


# ------------------------------------------------------------------------ GroupNorm at the VAE's group sizes ------
VAE_GN_EPS = 1e-6


@pytest.mark.gpu
@pytest.mark.parametrize("mu", (0, 8, 64))
@pytest.mark.parametrize("sigma", (1.0, 1e-3))
@pytest.mark.parametrize("b,hw,c", [(2, 262144, 128), (2, 65536, 256), (2, 4096, 512)])
def test_groupnorm_vae_statistics(b, hw, c, sigma, mu):
    """GroupNorm at eps 1e-6 over the VAE's groups (up to 4 channels x 512^2 pixels = 1 M elements) whose values sit at
    an offset of mu standard deviations, at sigma = 1 and at sigma = sqrt(eps) = 1e-3, where a variance that
    E[x^2] - E[x]^2 cancels to 0 in fp32 would give rstd = 1000 instead of ~707; from the slab statistics of the
    producing GEMM (8192 slabs per group at 512^2) and from the two-pass path"""
    be = Backend("cuda")
    g = torch.Generator().manual_seed(181)
    per_group = mu * sigma * torch.where(torch.arange(32) % 2 == 0, 1.0, -1.0) * (1 + 0.1 * torch.rand(32, generator=g))
    dc = per_group.repeat_interleave(c // 32).to(be.dev)
    x, st = _produce_unit(be, list(range(b)), hw, c, dc, sigma)
    sc = torch.ones(c, device=be.dev)
    bi = torch.zeros(c, device=be.dev)
    ref_fn = lambda v: _gn_ref(v, sc, bi, b, hw, False, VAE_GN_EPS)

    def f32_fn(v):
        t = v.reshape(b, hw, 32, c // 32)
        mean = t.mean(dim=(1, 3), keepdim=True)
        var = ((t * t).mean(dim=(1, 3), keepdim=True) - mean * mean).clamp(min=0)
        return ((t - mean) * torch.rsqrt(var + VAE_GN_EPS)).reshape(-1, c)

    e32 = _torch_f32_error(x, ref_fn, f32_fn)
    ref = ref_fn(x)
    for name, s0 in (("slab stats", st), ("two-pass", None)):
        got = _gn_launch(be, x, None, s0, None, sc, bi, b, hw, c, 0, False, ["y_f32", "y_bf16"], VAE_GN_EPS)
        _check_vs_f32(name + " y_f32", got["y_f32"], ref, e32, F32_MAX, F32_L2)
        _check_vs_f32(name + " y_bf16", got["y_bf16"], ref, e32, BF16_MAX, BF16_L2)


# ------------------------------------------------------------------------- the whole model against float64 ------
# Bounds at about twice the errors measured on an H100 80GB HBM3 (700 W power limit), which are in the comments; the
# ceiling on raw is the 3e-2 relative L2 the small configurations are held to (tests/test_gpu_z_vae.py).  bf16 operands
# through ~30 layers move about 0.8 % of the output, so about 40 % of the uint8 values land one level or more off the
# float64 image.
DECODE_RAW_L2 = 1.6e-2        # relative L2 of raw: 7.8e-3
DECODE_RAW_MAX = 1.5e-2       # max |error| / max |raw|: 7.4e-3
DECODE_U8_MAX = 8             # largest difference of the uint8 images, in levels: 4
DECODE_U8_SHARE = 0.5         # share of uint8 values that differ: 0.39
ENCODE_L2 = 1.3e-2            # relative L2 of the moments: 6.3e-3
ENCODE_MAX = 1.5e-2           # max |error| / max |moments|: 7.3e-3


def _rel(got, ref):
    d = got.double() - ref
    return (d.norm() / ref.norm()).item(), (d.abs().max() / ref.abs().max()).item()


@pytest.mark.gpu
def test_vae_decode_full_size_against_float64():
    """SD VAE decoder, three 64x64 latents -> 512x512 at decode_batch 2 (a chunk of 2 and a chunk of 1), against the
    oracle decoder in float64 on the GPU with the same parameters; the uint8 images the rewards consume; and the same
    bits at decode_batch 1"""
    from oracle import vae as OV
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    cfg = vae_mod.SD_VAE
    flat = vae_mod.init_flat_params(cfg, 0)
    lat = torch.randn(3, 4, 64, 64, generator=torch.Generator().manual_seed(5)) * vae_mod.VAE_SCALING
    dec = vae_mod.VAEDecoder(cfg, flat, "cuda", decode_batch=2)
    img, raw = dec.decode(lat.cuda(), want_raw=True, want_images=True)
    torch.cuda.synchronize()
    with torch.no_grad():
        img_r, raw_r = OV.decode(vae_mod.views(flat.cuda(), cfg), cfg, lat.cuda(), dtype=torch.float64)
    img_r = img_r.contiguous()
    l2, mx = _rel(raw, raw_r)
    u8, u8_r = (img * 255).to(torch.uint8), (img_r * 255).to(torch.uint8)
    du8 = (u8.int() - u8_r.int()).abs()
    u8_max, u8_share = du8.max().item(), (du8 > 0).double().mean().item()
    _record("decode raw", l2=l2, max=mx)
    _record("decode uint8", max=u8_max, share=u8_share)
    assert l2 <= DECODE_RAW_L2 and mx <= DECODE_RAW_MAX, f"raw: relative L2 {l2:.3g}, max {mx:.3g}"
    assert u8_max <= DECODE_U8_MAX and u8_share <= DECODE_U8_SHARE, f"uint8: max {u8_max}, share {u8_share:.3g}"
    dec.decode_batch = 1
    img1, raw1 = dec.decode(lat.cuda(), want_raw=True, want_images=True)
    torch.cuda.synchronize()
    for i in range(3):
        _same_bits(f"image {i} at decode_batch 1", img1[i], img[i])
        _same_bits(f"raw {i} at decode_batch 1", raw1[i], raw[i])


@pytest.mark.gpu
def test_vae_encode_full_size_against_float64():
    """SD VAE encoder, two 512x512 images -> 64x64x8 moments in one chunk, against the oracle encoder in float64 on the
    GPU"""
    from oracle import vae as OV
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    cfg = vae_mod.SD_VAE
    flat = vae_mod.init_flat_params(cfg, 2, part="encoder")
    img = torch.rand(2, 512, 512, 3, generator=torch.Generator().manual_seed(9))
    enc = vae_mod.VAEEncoder(cfg, flat, "cuda", decode_batch=2)
    mom = enc.encode(img.cuda())
    torch.cuda.synchronize()
    with torch.no_grad():
        ref = OV.encode(vae_mod.views(flat.cuda(), cfg, part="encoder"), cfg, img.cuda(), dtype=torch.float64)
    l2, mx = _rel(mom, ref)
    _record("encode moments", l2=l2, max=mx)
    assert l2 <= ENCODE_L2 and mx <= ENCODE_MAX, f"moments: relative L2 {l2:.3g}, max {mx:.3g}"
