"""Thin typed wrappers: torch tensors in -> C-ABI calls on the current CUDA stream.

torch is used for device memory and streams only; every arithmetic op below runs in
``libddpo_b200.so``.  Tensors must live on the current CUDA device.
"""
import ctypes as C

import numpy as np
import torch

from ._lib import AttentionArgs, AttentionBwdArgs, DdimCommon, GroupNormArgs, IGemmArgs, WgradArgs, check, lib

DDIM_CHUNKS = 8

# ---- instrumentation (bench.py): kernel-launch counter and optional CUDA-event profile ----
LAUNCH_COUNT = 0           # kernels launched through this module since import
PROFILE = None             # list of (name, work, event0, event1) while profiling, else None
PROFILE_TAGS = []          # parallel to PROFILE: a shape tag per entry (bench.py --shapes)
# kernels per call where it is not one; approximate (groupnorm_fwd launches one to three: statistics, finalize, apply)
_KERNELS_PER_CALL = {"groupnorm_fwd": 2, "groupnorm_bwd": 3, "layernorm_bwd": 2, "attention_bwd": 3, "colsum_cast": 2,
                     "conv_out_bwd": 3, "conv_in_wgrad": 2, "dense_small_bwd": 3, "grad_sumsq": 2, "wgrad": 2,
                     "colsum_bf16": 2, "clip_adafactor": 5, "lora_grad": 2}


def _launch(name, *args, work=0.0, tag="", symbol=None):
    """``ddpo_<symbol or name>(*args, stream)`` on the current stream: counts its kernels and checks its status.  While
    ``PROFILE`` is a list, CUDA events bracket the call, which is recorded as ``name`` with ``work`` and the shape tag
    ``tag`` (callers build a tag only while profiling)."""
    global LAUNCH_COUNT
    e0 = None
    if PROFILE is not None:
        e0 = torch.cuda.Event(enable_timing=True)
        e0.record()
    status = getattr(lib(), "ddpo_" + (symbol or name))(*args, _stream())
    LAUNCH_COUNT += _KERNELS_PER_CALL.get(name, 1)
    if e0 is not None:
        e1 = torch.cuda.Event(enable_timing=True)
        e1.record()
        PROFILE.append((name, work, e0, e1))
        PROFILE_TAGS.append(tag)
    check(status, name)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    if t is None:
        return None
    assert t.is_cuda, "ddpo_b200 ops need CUDA tensors (no CPU fallback)"
    return C.c_void_p(t.data_ptr())


def _chk(t, dtype, name):
    assert t.is_cuda and t.dtype == dtype and t.is_contiguous(), f"{name}: need contiguous CUDA {dtype}, got {t.dtype} {t.device}"


# ---- scratch workspaces of the kernels that plan their own (wgrad, colsum, stems, LoRA), grown on demand ----
# kind -> device -> fp32 tensor
_WORKSPACES = {kind: {} for kind in ("wgrad", "colsum", "conv_out_bwd", "conv_in_wgrad", "lora_grad")}
_WGRAD_WS = _WORKSPACES["wgrad"]   # the wgrad tests swap a workspace of their own in here


def _workspace(kind, device, need, min_floats=1 << 20):
    """The fp32 workspace of ``kind`` on ``device``: at least ``need`` floats.  One that is too small is replaced by
    a new one of max(need, min_floats) floats; a CUDA graph captured with the old one keeps it (``graph_step``)."""
    cache = _WORKSPACES[kind]
    ws = cache.get(device)
    if ws is None or ws.numel() < need:
        ws = cache[device] = torch.empty(max(need, min_floats), dtype=torch.float32, device=device)
    return ws


def graph_step(captured, sig, body, enabled, protect=None):
    """Run ``body()``, one step of kernels on fixed buffers, as the replay of a CUDA graph (eagerly when not
    ``enabled``).  ``captured`` is what the previous call for these buffers returned, None at first.  Without a graph,
    or with one captured at another ``sig``, the body first runs eagerly (the warm-up grows the arena and the
    workspaces and sets kernel attributes; ``protect``, e.g. a gradient accumulator, gets its contents back after it)
    and is then captured.

    Returns what to pass next time: the signature, the graph and the workspaces it was captured with.  Holding those
    keeps a workspace that ``_workspace`` has since replaced alive exactly as long as a graph that writes to it."""
    if not enabled:
        body()
        return captured
    if captured is None or captured[0] != sig:
        saved = protect.clone() if protect is not None else None
        body()
        torch.cuda.synchronize()
        if protect is not None:
            protect.copy_(saved)
        del saved   # a full gradient copy: freed before the capture allocates
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            body()
        captured = (sig, graph, [ws for cache in _WORKSPACES.values() for ws in cache.values()])
    captured[1].replay()
    return captured


# ------------------------------------------------------------------ PRNG --------
def prng_key(seed: int):
    out = (C.c_uint32 * 2)()
    check(lib().ddpo_prng_key_host(C.c_uint64(seed & (2 ** 64 - 1)), out), "prng_key")
    return (int(out[0]), int(out[1]))


def threefry_split(key, num=2):
    k = (C.c_uint32 * 2)(key[0], key[1])
    out = (C.c_uint32 * (2 * num))()
    check(lib().ddpo_threefry_split_host(k, num, out), "threefry_split")
    return [(int(out[2 * i]), int(out[2 * i + 1])) for i in range(num)]


def threefry_randint(key, n, minval, maxval):
    """jax.random.randint(key, (n,), minval, maxval) on the host -> list of ints."""
    k = (C.c_uint32 * 2)(key[0], key[1])
    out = (C.c_int32 * int(n))()
    check(lib().ddpo_threefry_randint_host(k, int(n), int(minval), int(maxval), out), "threefry_randint")
    return [int(v) for v in out]


def key_tensor(keys, device):
    """[(k0,k1), ...] -> int64-free uint32 storage as int32 tensor [len, 2] on device."""
    flat = []
    for k in keys:
        flat += [k[0] if k[0] < 2 ** 31 else k[0] - 2 ** 32, k[1] if k[1] < 2 ** 31 else k[1] - 2 ** 32]
    return torch.tensor(flat, dtype=torch.int32).view(-1, 2).to(device)


def threefry_normal(key_dev, out):
    _chk(out, torch.float32, "out")
    _launch("threefry_normal", _p(key_dev), _p(out), out.numel())
    return out


# ------------------------------------------------------------------ DDIM --------
def ddim_workspace(batch, device):
    return torch.zeros(batch * DDIM_CHUNKS + batch, dtype=torch.float32, device=device)


PREDICTION_TYPES = {"epsilon": 0, "sample": 1, "v_prediction": 2}   # scheduling_ddim_flax.py:303-321


def prediction_code(prediction_type):
    """FlaxDDIMScheduler's config string -> the C ABI's DDPO_PRED_* code; same ValueError text as the reference (:317-321)."""
    if prediction_type not in PREDICTION_TYPES:
        raise ValueError(f"prediction_type given as {prediction_type} must be one of `epsilon`, `sample`, or"
                         " `v_prediction`")
    return PREDICTION_TYPES[prediction_type]


def _ddim_common(eps_u, eps_c, sample, alphas_cumprod, timesteps, final_alpha, step_ratio, guidance, eta, ws,
                 pred="epsilon"):
    b = sample.shape[0]
    n = sample.numel() // b
    for t, nm in ((eps_u, "eps_u"), (eps_c, "eps_c"), (sample, "sample"), (alphas_cumprod, "alphas_cumprod")):
        _chk(t, torch.float32, nm)
    _chk(timesteps, torch.int32, "timesteps")
    assert timesteps.numel() in (1, b)
    c = DdimCommon(_p(eps_u), _p(eps_c), _p(sample), _p(alphas_cumprod), _p(timesteps),
                   1 if timesteps.numel() == b and b > 1 else (0 if timesteps.numel() == 1 else 1),
                   float(final_alpha), int(step_ratio), float(guidance), float(eta), b, n, _p(ws), prediction_code(pred))
    return c


def ddim_step_sample(eps_u, eps_c, sample, alphas_cumprod, timesteps, final_alpha, step_ratio, guidance, eta,
                     key_dev, prev_out, logp_out, ws, pred="epsilon"):
    c = _ddim_common(eps_u, eps_c, sample, alphas_cumprod, timesteps, final_alpha, step_ratio, guidance, eta, ws, pred)
    _launch("ddim_step_sample", C.byref(c), _p(key_dev), _p(prev_out), _p(logp_out))


def ddim_logprob_fwd(eps_u, eps_c, sample, prev, alphas_cumprod, timesteps, final_alpha, step_ratio, guidance, eta,
                     logp_out, ws, pred="epsilon"):
    c = _ddim_common(eps_u, eps_c, sample, alphas_cumprod, timesteps, final_alpha, step_ratio, guidance, eta, ws, pred)
    _launch("ddim_logprob_fwd", C.byref(c), _p(prev), _p(logp_out))


def ddim_logprob_bwd(eps_u, eps_c, sample, prev, alphas_cumprod, timesteps, final_alpha, step_ratio, guidance, eta,
                     dlogp, d_eps_u, d_eps_c, ws, pred="epsilon"):
    c = _ddim_common(eps_u, eps_c, sample, alphas_cumprod, timesteps, final_alpha, step_ratio, guidance, eta, ws, pred)
    _launch("ddim_logprob_bwd", C.byref(c), _p(prev), _p(dlogp), _p(d_eps_u), _p(d_eps_c))


def ppo_loss(logp, old_logp, adv, clip_range, info_out, dlogp_out, micro_batch=None):
    _launch("ppo_loss", _p(logp), _p(old_logp), _p(adv), logp.numel(), int(micro_batch or logp.numel()), float(clip_range),
            _p(info_out), _p(dlogp_out))


# ------------------------------------------------------------------ GEMM --------
def igemm(*, a0, wt, n, a1=None, c0=None, c1=0, lda0=None, lda1=None, conv=None, m=None, taps=1, stride=1,
          bias=None, rowvec=None, rows_per_sample=0, rowvec_ld=0, residual=None, ld_res=0, out_f32=None,
          out_bf16=None, ld_out=0, geglu=False, accumulate=False, bn=0, aux_bf16=None, gn_stats=None,
          no_low_pad=False, bm=0):
    """conv=(batch, h_out, w_out) for convolutions, else linear with m rows.  ``bm`` / ``bn`` force the output tile's
    height / width (tests; 0 = the library's plan, ``igemm_plan``)."""
    a = IGemmArgs()
    a.a0, a.a1 = _p(a0), _p(a1)
    a.c0 = int(c0 if c0 is not None else a0.shape[-1])
    a.c1 = int(c1)
    a.lda0 = int(lda0 if lda0 is not None else a.c0)
    a.lda1 = int(lda1 if lda1 is not None else a.c1)
    if conv is not None:
        a.is_conv, a.batch, a.h, a.w = 1, int(conv[0]), int(conv[1]), int(conv[2])
        a.m = 0
    else:
        a.is_conv, a.batch, a.h, a.w = 0, 0, 0, 0
        a.m = int(m)
    a.conv_stride, a.taps, a.n = int(stride), int(taps), int(n)
    a.wt, a.bias, a.rowvec = _p(wt), _p(bias), _p(rowvec)
    a.rows_per_sample, a.rowvec_ld = int(rows_per_sample), int(rowvec_ld)
    a.residual, a.ld_res = _p(residual), int(ld_res)
    a.out_f32, a.out_bf16, a.ld_out = _p(out_f32), _p(out_bf16), int(ld_out)
    a.geglu, a.accumulate_out, a.bn_override = int(geglu), int(accumulate), int(bn)
    a.aux_bf16 = _p(aux_bf16)
    a.gn_stats = _p(gn_stats)
    a.conv_pad = int(no_low_pad)
    a.bm_override = int(bm)
    rows = a.batch * a.h * a.w if a.is_conv else a.m
    _launch("igemm", C.byref(a), work=2.0 * rows * a.n * a.taps * (a.c0 + a.c1),
            tag=f"M{rows} N{a.n} K{a.taps * (a.c0 + a.c1)} taps{a.taps} s{a.conv_stride}"
                f"{' geglu' if geglu else ''}{' res' if residual is not None else ''}"
                f"{' f32' if out_f32 is not None else ''}{' bf16' if out_bf16 is not None else ''}"
                f"{' acc' if accumulate else ''}" if PROFILE is not None else "")


def igemm_plan(m, n, k, geglu=False, bm=0, bn=0):
    """(BM, BN, CTAs per SM, operand stages) of the tile ``igemm`` runs for an [m, k] x [k, n] product; host only."""
    plan = (C.c_int * 4)()
    check(lib().ddpo_igemm_plan(int(m), int(n), int(k), int(geglu), int(bm), int(bn), plan), "igemm_plan")
    return tuple(plan)


# ------------------------------------------------------------------ norms -------
def groupnorm_workspace_floats(batch, hw, channels):
    return int(lib().ddpo_groupnorm_workspace_floats(batch, hw, channels))


def _gn_args(x0, x1, c0, c1, batch, hw, scale, bias, silu, y_bf16, y_f32, raw_bf16, ws, ld0=0, ld1=0, skip_stats=False,
             eps=1e-5, stats0=None, stats1=None, dy_bf16=False):
    return GroupNormArgs(_p(x0), _p(x1), int(c0), int(c1), int(ld0), int(ld1), int(batch), int(hw), _p(scale),
                         _p(bias), float(eps), int(silu), _p(y_bf16), _p(y_f32), _p(raw_bf16), _p(ws), int(skip_stats),
                         _p(stats0), _p(stats1), int(dy_bf16))


def gn_stats_shape(rows, channels):
    """Shape of the slab-statistics buffer an igemm with ``gn_stats=`` fills for its [rows, channels] fp32 output."""
    return ((int(rows) + 31) // 32, int(channels), 2)


def groupnorm_fwd(x0, scale, bias, ws, batch, hw, c0, x1=None, c1=0, silu=True, y_bf16=None, y_f32=None,
                  raw_bf16=None, skip_stats=False, eps=1e-5, stats0=None, stats1=None):
    """``stats0`` / ``stats1``: slab statistics of x0 / x1 left by the igemm that produced them (``gn_stats=``); with both
    (or ``stats0`` alone for one source) and hw % 32 == 0 the statistics pass over x is skipped."""
    a = _gn_args(x0, x1, c0, c1, batch, hw, scale, bias, silu, y_bf16, y_f32, raw_bf16, ws, skip_stats=skip_stats,
                 eps=eps, stats0=stats0, stats1=stats1)
    per = 4 + (2 if y_bf16 is not None else 0) + (4 if y_f32 is not None else 0) + (2 if raw_bf16 is not None else 0)
    _launch("groupnorm_fwd", C.byref(a), work=float(batch) * hw * (c0 + c1) * per)


def groupnorm_bwd(x0, scale, bias, ws, batch, hw, c0, dy, dx0, dscale, dbias, x1=None, c1=0, dx1=None, silu=True,
                  accumulate=False, ldd0=0, ldd1=0):
    """``dy`` fp32 or bf16 (the dtype selects the kernel's load path): the dgrad GEMM in front of a GroupNorm writes bf16."""
    assert dy.dtype in (torch.float32, torch.bfloat16)
    a = _gn_args(x0, x1, c0, c1, batch, hw, scale, bias, silu, None, None, None, ws, dy_bf16=dy.dtype == torch.bfloat16)
    _launch("groupnorm_bwd", C.byref(a), _p(dy), _p(dx0), _p(dx1), int(ldd0), int(ldd1), int(accumulate), _p(dscale),
            _p(dbias))


def layernorm_fwd(x, scale, bias, y_bf16, m, c, stats=None):
    _launch("layernorm_fwd", _p(x), _p(scale), _p(bias), _p(y_bf16), _p(stats), int(m), int(c), 1e-5)


def layernorm_bwd_workspace_floats(m, c):
    return int(lib().ddpo_layernorm_bwd_workspace_floats(m, c))


def layernorm_bwd(x, scale, stats, dy, dx, dscale, dbias, ws, m, c, accumulate=False):
    assert dy.dtype in (torch.float32, torch.bfloat16)
    _launch("layernorm_bwd", _p(x), _p(scale), _p(stats), _p(dy), _p(dx), int(accumulate), _p(dscale), _p(dbias), _p(ws),
            int(m), int(c), int(dy.dtype == torch.bfloat16))


# ------------------------------------------------------------ small layers -------
def prep_weight(src, dst, k, n, ldk=None, row_offset=0, col_offset=0, geglu_bn=0):
    _launch("prep_weight", _p(src), _p(dst), int(k), int(n), int(ldk or k), int(row_offset), int(col_offset),
            int(geglu_bn))


def prep_weight_dgrad(src, dst, taps, k, n, ld_dst=0, col_offset=0):
    _launch("prep_weight_dgrad", _p(src), _p(dst), int(taps), int(k), int(n), int(ld_dst), int(col_offset))


def permute_geglu_bias(src, dst, n, bn):
    _launch("permute_geglu_bias", _p(src), _p(dst), int(n), int(bn))


def cast_bf16(x, y):
    _launch("cast_bf16", _p(x), _p(y), x.numel())


def upsample2x_bf16(x, y, batch, h, w, c):
    _launch("upsample2x_bf16", _p(x), _p(y), batch, h, w, c)


def upsample2x_bwd(dy, dx, batch, h, w, c, accumulate=False):
    _launch("upsample2x_bwd", _p(dy), _p(dx), batch, h, w, c, int(accumulate))


def conv_in(x_nchw, w, bias, y_nhwc, batch, cin, h, wd, cout, gn_stats=None):
    _launch("conv_in", _p(x_nchw), _p(w), _p(bias), _p(y_nhwc), batch, cin, h, wd, cout, _p(gn_stats))


def conv_out(x_nhwc, w, bias, y_nchw, batch, h, wd, cin, cout):
    _launch("conv_out", _p(x_nhwc), _p(w), _p(bias), _p(y_nchw), batch, h, wd, cin, cout)


def timestep_sincos(t, out, batch, dim):
    _launch("timestep_sincos", _p(t), 1 if t.numel() > 1 else 0, _p(out), batch, dim)


def dense_small(x, w, bias, y, batch, k, n, silu_in=False, silu_out=False):
    _launch("dense_small", _p(x), _p(w), _p(bias), _p(y), batch, k, n, int(silu_in), int(silu_out))


def dense_small_group_table(entries, device):
    """entries: [(w_off, bias_off, y_off, n)] in floats -> (device uint8 table, total CTAs) for dense_small_grouped."""
    rec = np.zeros(len(entries), dtype=[("w", "<i8"), ("b", "<i8"), ("y", "<i8"), ("n", "<i4"), ("cta0", "<i4")])
    cta = 0
    for i, (w_off, b_off, y_off, n) in enumerate(entries):
        rec[i] = (w_off, b_off, y_off, n, cta)
        cta += (n + 31) // 32
    return torch.from_numpy(rec.view(np.uint8).copy()).to(device), cta


def dense_small_grouped(x, params_base, y_base, table, n_groups, total_ctas, batch, k):
    _launch("dense_small", _p(x), _p(params_base), _p(y_base), _p(table), int(n_groups), int(total_ctas), int(batch),
            int(k), symbol="dense_small_grouped")


# --------------------------------------------------------------- attention -------
ATTENTION_HEAD_DIMS = (40, 64, 80, 160)   # what ddpo_attention_fwd / _bwd accept (SD2: 64; SD1.x: 40, 80, 160)


def attention_fwd(q, k, v, out, batch, heads, nq, nk, ldq, ldk, ldv, ldo, lse=None, causal=False, head_dim=64):
    """head h of q/k/v/out at columns [h * head_dim, (h + 1) * head_dim); head_dim is 40, 64, 80 or 160"""
    a = AttentionArgs(_p(q), _p(k), _p(v), _p(out), _p(lse), batch, heads, nq, nk, head_dim, ldq, ldk, ldv, ldo,
                      int(causal))
    _launch("attention_fwd", C.byref(a), work=4.0 * batch * heads * nq * nk * head_dim,
            tag=f"B{batch} H{heads} nq{nq} nk{nk}" if PROFILE is not None else "")


# ------------------------------------------------------------------ wgrad -------
def wgrad(*, dy, n, x0, dw, x1=None, c0=None, c1=0, ldy=0, ldx0=0, ldx1=0, conv=None, m=None, taps=1, stride=1,
          bn=0, splits=0):
    """dw[(tap, cin), n] += X^T dY (fp32, Flax layout).  conv=(batch, h_out, w_out) or linear with m rows.  ``bn`` /
    ``splits`` force the column-tile width / pixel split count (tests; 0 = the library's plan, ``wgrad_plan``)."""
    a = WgradArgs()
    a.dy, a.ldy, a.n = _p(dy), int(ldy), int(n)
    a.x0, a.x1 = _p(x0), _p(x1)
    a.c0 = int(c0 if c0 is not None else x0.shape[-1])
    a.c1, a.ldx0, a.ldx1 = int(c1), int(ldx0), int(ldx1)
    if conv is not None:
        a.is_conv, a.batch, a.h, a.w, a.m = 1, int(conv[0]), int(conv[1]), int(conv[2]), 0
    else:
        a.is_conv, a.batch, a.h, a.w, a.m = 0, 0, 0, 0, int(m)
    a.conv_stride, a.taps = int(stride), int(taps)
    a.dw = _p(dw)
    a.bn_override, a.splits_override = int(bn), int(splits)
    need = int(lib().ddpo_wgrad_workspace_floats(C.byref(a)))
    ws = _workspace("wgrad", dw.device, need) if need > 0 else None
    a.workspace = _p(ws)
    a.workspace_floats = ws.numel() if ws is not None else 0
    rows = a.batch * a.h * a.w if a.is_conv else a.m
    _launch("wgrad", C.byref(a), work=2.0 * rows * a.n * a.taps * (a.c0 + a.c1),
            tag=f"M{rows} N{a.n} K{a.taps * (a.c0 + a.c1)} taps{a.taps} s{a.conv_stride}" if PROFILE is not None else "")


def wgrad_plan(m, c0, n, c1=0, taps=1, bn=0, splits=0):
    """(BN, pixel splits) of the launch ``wgrad`` runs over m pixels (b*h*w of dY for convolutions); host only."""
    plan = (C.c_int * 2)()
    check(lib().ddpo_wgrad_plan(int(m), int(c0), int(c1), int(n), int(taps), int(bn), int(splits), plan), "wgrad_plan")
    return tuple(plan)


# ------------------------------------------------------- backward wrappers -------
def attention_bwd(q, k, v, out, dout, lse, delta, dq, dk, dv, batch, heads, nq, nk, ldq, ldk, ldv, ldo, lddo, lddq,
                  lddk, lddv, head_dim=64):
    a = AttentionBwdArgs(_p(q), _p(k), _p(v), _p(out), _p(dout), _p(lse), _p(delta), _p(dq), _p(dk), _p(dv), batch,
                         heads, nq, nk, head_dim, ldq, ldk, ldv, ldo, lddo, lddq, lddk, lddv)
    _launch("attention_bwd", C.byref(a), work=14.0 * batch * heads * nq * nk * head_dim,
            tag=f"B{batch} H{heads} nq{nq} nk{nk}" if PROFILE is not None else "")


def colsum_cast(dy, m, n, y_bf16=None, out=None, rows_per_group=None, accumulate=True, ld=0):
    """Optional bf16 copy of dy [m, n] and out[g, n] (+)= per-group column sums (bias / per-sample grads)."""
    rpg = int(rows_per_group or m)
    ws = None
    if out is not None:
        ws = _workspace("colsum", dy.device, int(lib().ddpo_colsum_workspace_floats(m, n, rpg)))
    _launch("colsum_cast", _p(dy), int(ld), _p(y_bf16), _p(out), rpg, int(accumulate), _p(ws), int(m), int(n),
            work=float(m) * n * 6)


def colsum_bf16(x, m, n, out, accumulate=True, ld=0):
    ws = _workspace("colsum", x.device, int(lib().ddpo_colsum_workspace_floats(m, n, m)))
    _launch("colsum_bf16", _p(x), int(ld), _p(out), int(accumulate), _p(ws), int(m), int(n), work=float(m) * n * 2)


def geglu_bwd(pre, dff, dpre, m, n, bn=256):
    assert dff.dtype in (torch.float32, torch.bfloat16)
    _launch("geglu_bwd", _p(pre), _p(dff), _p(dpre), int(m), int(n), int(bn), int(dff.dtype == torch.bfloat16))


def conv_out_bwd(x_nhwc, w, dy_nchw, dx_nhwc, dw, dbias, batch, h, wd, cin):
    ws = _workspace("conv_out_bwd", dw.device, int(lib().ddpo_conv_out_bwd_workspace_floats(cin)), min_floats=0)
    _launch("conv_out_bwd", _p(x_nhwc), _p(w), _p(dy_nchw), _p(dx_nhwc), _p(dw), _p(dbias), _p(ws), batch, h, wd, cin)


def conv_in_wgrad(lat, dx_nhwc, dw, batch, cin, h, wd, cout):
    ws = _workspace("conv_in_wgrad", dw.device, int(lib().ddpo_conv_in_wgrad_workspace_floats(cin, cout)), min_floats=0)
    _launch("conv_in_wgrad", _p(lat), _p(dx_nhwc), _p(dw), _p(ws), batch, cin, h, wd, cout)


def dense_small_bwd(x, w, bias, dy, dpre_ws, dw, db, dx, batch, k, n, silu_in=False, silu_out=False, dx_accumulate=False):
    _launch("dense_small_bwd", _p(x), _p(w), _p(bias), _p(dy), _p(dpre_ws), _p(dw), _p(db), _p(dx), int(dx_accumulate),
            batch, k, n, int(silu_in), int(silu_out))


def dilate2x_bf16(x, y, batch, h, w, c):
    _launch("dilate2x_bf16", _p(x), _p(y), batch, h, w, c)


def copy2d(src, lds, dst, ldd, rows, cols, accumulate=False):
    _launch("copy2d", _p(src), int(lds), _p(dst), int(ldd), int(rows), int(cols), int(accumulate))


def gather_rows(src, index, dst):
    """dst[r] = src[index[r]] for fp32 [rows, row_floats] matrices; index int64 on the device."""
    _chk(src, torch.float32, "src")
    _chk(dst, torch.float32, "dst")
    _chk(index, torch.int64, "index")
    rows = index.numel()
    row_floats = dst.numel() // rows
    assert src.numel() % row_floats == 0 and dst.numel() == rows * row_floats
    _launch("gather_rows", _p(src), _p(index), _p(dst), rows, row_floats, work=float(rows) * row_floats * 8)


def optim_workspace(device):
    return torch.empty(int(lib().ddpo_optim_workspace_bytes()), dtype=torch.uint8, device=device)


def grad_sumsq(g, ws, out):
    _launch("grad_sumsq", _p(g), g.numel(), _p(ws), _p(out), work=float(g.numel()) * 4)


def clip_adamw(params, grad_acc, mu, nu, sumsq, grad_scale, max_norm, lr, b1, b2, eps, wd, step, norm_out=None):
    _launch("clip_adamw", _p(params), _p(grad_acc), _p(mu), _p(nu), params.numel(), _p(sumsq), float(grad_scale),
            float(max_norm), float(lr), float(b1), float(b2), float(eps), float(wd), int(step), _p(norm_out),
            work=float(params.numel()) * 24)


class AdafactorPlan:
    """Output of the host planner ``ddpo_adafactor_plan``: which tensors are factored, the layout of the Adafactor
    state (optax's ``v_row``/``v_col``/``v``, leaf by leaf, in tensor order) and the tiling of the flat buffer.
    ``host`` is the plan as int64 words; ``tensors`` [T, 12] and ``tiles`` [L, 9] are views of its records (field
    order in ``csrc/adafactor.cu``)."""
    T_WORDS, L_WORDS = 12, 9

    def __init__(self, host, info, shapes, n, state_floats, workspace_floats):
        self.host, self.shapes, self.n = host, shapes, n
        self.state_floats, self.workspace_floats = state_floats, workspace_floats
        self.kinds = [int(k) for k in info[:, 0]]          # 0 unfactored, 1 v_row over dim -2, 2 v_row over dim -1
        self.state_offsets = [(int(a), int(b)) for a, b in info[:, 1:]]
        nt, nl = int(host[2]), int(host[3])
        self.tensors = host[8:8 + nt * self.T_WORDS].reshape(nt, self.T_WORDS)
        self.tiles = host[8 + nt * self.T_WORDS:8 + nt * self.T_WORDS + nl * self.L_WORDS].reshape(nl, self.L_WORDS)
        self._dev = {}

    def device_copy(self, device):
        d = self._dev.get(device)
        if d is None:
            d = self._dev[device] = torch.from_numpy(self.host).to(device)
        return d

    def state_shapes(self, t):
        """optax's state leaves of tensor t: {"v_row": shape, "v_col": shape} or {"v": shape}"""
        s, k = tuple(self.shapes[t]), self.kinds[t]
        if k == 0:
            return {"v": s}
        over_rows, over_cols = s[:-1], s[:-2] + s[-1:]
        return {"v_row": over_rows, "v_col": over_cols} if k == 1 else {"v_row": over_cols, "v_col": over_rows}

    def state_views(self, state):
        """per tensor, the views of the flat state buffer named as optax names them"""
        out = []
        for t in range(len(self.shapes)):
            d = {}
            for (name, shape), off in zip(self.state_shapes(t).items(), self.state_offsets[t]):
                d[name] = state[off:off + int(np.prod(shape))].view(*shape)
            out.append(d)
        return out


def adafactor_plan(tensors, n, min_dim_size_to_factor=128):
    """Host-only planner.  ``tensors``: [(offset, shape)] views of the flat n-float buffer, ascending offsets."""
    offs = np.array([int(o) for o, _ in tensors], np.int64)
    nd = np.array([len(s) for _, s in tensors], np.int32)
    dims = np.array([int(d) for _, s in tensors for d in s], np.int64)
    sizes = np.zeros(3, np.int64)
    info = np.zeros((len(tensors), 3), np.int64)
    args = (len(tensors), offs.ctypes.data, nd.ctypes.data, dims.ctypes.data, int(n), int(min_dim_size_to_factor))
    check(lib().ddpo_adafactor_plan(*args, None, 0, sizes.ctypes.data, None), "adafactor_plan")
    host = np.zeros(int(sizes[0]), np.int64)
    check(lib().ddpo_adafactor_plan(*args, host.ctypes.data, host.size, sizes.ctypes.data, info.ctypes.data),
          "adafactor_plan")
    return AdafactorPlan(host, info, [tuple(int(d) for d in s) for _, s in tensors], int(n), int(sizes[1]), int(sizes[2]))


def clip_adafactor(params, grad_acc, state, plan, workspace, sumsq, grad_scale, max_norm, lr, wd, step, norm_out=None):
    for t, nm in ((params, "params"), (grad_acc, "grad_acc"), (state, "state"), (workspace, "workspace")):
        _chk(t, torch.float32, nm)
    assert grad_acc.numel() == params.numel()
    _launch("clip_adafactor", _p(params), _p(grad_acc), _p(state), state.numel(), params.numel(), plan.host.ctypes.data,
            _p(plan.device_copy(params.device)), _p(workspace), workspace.numel(), _p(sumsq), float(grad_scale),
            float(max_norm), float(lr), float(wd), int(step), _p(norm_out), work=float(params.numel()) * 28)


# --------------------------------------------------------------------- RWR -------
def rwr_workspace(batch, device):
    return torch.zeros(int(lib().ddpo_rwr_workspace_floats(int(batch))), dtype=torch.float32, device=device)


def rwr_noisy_latents(moments_nhwc, key_sample_dev, key_noise_dev, timesteps, alphas_cumprod, noise_out, noisy_out,
                      latents_out=None, scaling=0.18215):
    """moments [B,h,w,2C] fp32 -> noise / noisy latents [B,C,h,w] (reference ddpo/training/diffusion.py:16-43)."""
    _chk(moments_nhwc, torch.float32, "moments")
    _chk(timesteps, torch.int32, "timesteps")
    _chk(noise_out, torch.float32, "noise_out")
    _chk(noisy_out, torch.float32, "noisy_out")
    b, h, w, c2 = moments_nhwc.shape
    assert timesteps.numel() == b and noise_out.numel() == b * (c2 // 2) * h * w == noisy_out.numel()
    _launch("rwr_noisy_latents", _p(moments_nhwc), _p(key_sample_dev), _p(key_noise_dev), _p(timesteps),
            _p(alphas_cumprod), float(scaling), b, c2 // 2, h, w, _p(noise_out), _p(noisy_out), _p(latents_out))


def rwr_mse_loss(eps_u, eps_c, noise, guidance, loss_out, ws, weights=None, per_sample=None, d_eps_u=None, d_eps_c=None):
    """loss of ddpo/training/diffusion.py:77-90 and its gradient wrt both U-Net outputs; eps_* / noise are [B, n]."""
    for t, nm in ((eps_u, "eps_u"), (eps_c, "eps_c"), (noise, "noise")):
        _chk(t, torch.float32, nm)
    b = noise.shape[0]
    n = noise.numel() // b
    if weights is not None:
        _chk(weights, torch.float32, "weights")
        assert weights.numel() == b
    _launch("rwr_mse_loss", _p(eps_u), _p(eps_c), _p(noise), _p(weights), float(guidance), b, n, _p(loss_out),
            _p(per_sample), _p(d_eps_u), _p(d_eps_c), _p(ws))


# --------------------------------------------------------------------- VAE -------
def vae_post_quant(latents, w, bias, out, scaling=0.18215):
    _chk(latents, torch.float32, "latents")
    _chk(out, torch.float32, "out")
    b, c, h, wd = latents.shape
    _launch("vae_post_quant", _p(latents), _p(w), _p(bias), float(scaling), b, c, h, wd, _p(out))


def softmax_rows(scores, probs_bf16, scale):
    """probs[r] = softmax(scale * scores[r]); scores fp32 [rows, n], probs bf16 [rows, n] (row-contiguous)."""
    _chk(scores, torch.float32, "scores")
    _chk(probs_bf16, torch.bfloat16, "probs")
    rows, n = scores.shape
    _launch("softmax_rows", _p(scores), n, float(scale), _p(probs_bf16), n, rows, n, work=float(rows) * n * 6)


def image_to_uint8(img, out_u8):
    """``(img * 255).astype(uint8)`` (the reference's truncating cast, callbacks.py:181) on the device"""
    _chk(img, torch.float32, "images")
    _chk(out_u8, torch.uint8, "out")
    assert img.numel() == out_u8.numel() and img.numel() % 4 == 0
    _launch("image_to_uint8", _p(img), _p(out_u8), img.numel())


# ------------------------------------------------- image-symmetry / consistency rewards -------
def resample_u8(src, transform, axis, table_host, table_dev, dst):
    """one pass of Pillow's bicubic resize (``include/ddpo_b200.h``); ``table_host`` int32 numpy and ``table_dev`` its
    device copy (``clip_vision.resample_table``)"""
    _chk(src, torch.uint8, "src")
    _chk(dst, torch.uint8, "dst")
    _chk(table_dev, torch.int32, "table")
    assert table_host.dtype == np.int32 and table_host.flags.c_contiguous and tuple(table_dev.shape) == table_host.shape
    b, h, w, c = src.shape
    n_out = table_host.shape[0]
    th, tw = (w, h) if transform in (2, 4) else (h, w)
    assert c == 3 and tuple(dst.shape) == ((b, th, n_out, 3) if axis == 0 else (b, n_out, tw, 3)), (src.shape, dst.shape)
    _launch("resample_u8", _p(src), b, h, w, int(transform), int(axis), n_out, table_host.ctypes.data, _p(table_dev),
            table_host.shape[1] - 2, _p(dst), work=float(dst.numel() + src.numel()))


def clip_normalize_u8(src, top, left, out):
    """CLIP rescale + normalise of the ``size`` x ``size`` crop at (top, left) -> fp32 NHWC ``out``"""
    _chk(src, torch.uint8, "src")
    _chk(out, torch.float32, "out")
    b, h, w, _ = src.shape
    size = out.shape[1]
    assert tuple(out.shape) == (b, size, size, 3)
    _launch("clip_normalize_u8", _p(src), b, h, w, int(top), int(left), size, _p(out), work=float(out.numel()) * 5)


def pair_stats_u8(src, transform, out):
    """per image against its mirror (1) or 180-degree rotation (3): int64 [B, 4] = (sum of uint8-wrapped squared
    differences, sum a, sum a^2, sum a T(a))"""
    _chk(src, torch.uint8, "src")
    _chk(out, torch.int64, "out")
    b, h, w, _ = src.shape
    assert tuple(out.shape) == (b, 4)
    _launch("pair_stats_u8", _p(src), b, h, w, int(transform), _p(out), work=float(src.numel()) * 2)


def feature_angles(feats, variants, out):
    """feats fp32 [variants * n, dim] -> out [n]: mean over variants >= 1 of the angle (degrees) to variant 0"""
    _chk(feats, torch.float32, "feats")
    _chk(out, torch.float32, "out")
    n = out.numel()
    assert feats.dim() == 2 and feats.shape[0] == variants * n
    _launch("feature_angles", _p(feats), int(variants), n, feats.shape[1], _p(out), work=float(feats.numel()) * 4)


def scaled_cosine(img, txt, logit_scale, out):
    """out[i] = exp(logit_scale) cos(img[i], txt[i])"""
    _chk(img, torch.float32, "img")
    _chk(txt, torch.float32, "txt")
    _chk(out, torch.float32, "out")
    assert img.shape == txt.shape and img.dim() == 2 and out.numel() == img.shape[0]
    _launch("scaled_cosine", _p(img), _p(txt), img.shape[0], img.shape[1], float(logit_scale), _p(out),
            work=float(img.numel()) * 8)


def vae_image_to_nchw(img_nhwc, out_nchw):
    _chk(img_nhwc, torch.float32, "images")
    _chk(out_nchw, torch.float32, "out")
    b, h, w, c = img_nhwc.shape
    assert c == 3 and tuple(out_nchw.shape) == (b, 3, h, w)
    _launch("vae_image_to_nchw", _p(img_nhwc), _p(out_nchw), b, h, w)


def vae_encoder_head(x_nhwc, w, bias, wq, bq, moments, batch, h, wd, cin):
    _chk(moments, torch.float32, "moments")
    _launch("vae_encoder_head", _p(x_nhwc), _p(w), _p(bias), _p(wq), _p(bq), _p(moments), batch, h, wd, cin)


def vae_conv_out(x_nhwc, w, bias, batch, h, wd, cin, raw_nchw=None, img_nhwc=None):
    _launch("vae_conv_out", _p(x_nhwc), _p(w), _p(bias), _p(raw_nchw), _p(img_nhwc), batch, h, wd, cin)


# ------------------------------------------------------------ text encoder -------
def embed_tokens(ids, token_embedding, position_embedding, out, seq_len):
    _chk(ids, torch.int32, "ids")
    _chk(out, torch.float32, "out")
    rows, dim = out.shape
    _launch("embed_tokens", _p(ids), _p(token_embedding), _p(position_embedding), _p(out), rows, int(seq_len), dim,
            token_embedding.shape[0])


def act_bf16(x, y_bf16, act):
    """act: "gelu" (erf form) or "quick_gelu"."""
    _chk(x, torch.float32, "x")
    _chk(y_bf16, torch.bfloat16, "y")
    _launch("act_bf16", _p(x), _p(y_bf16), x.numel(), {"gelu": 0, "quick_gelu": 1}[act], work=float(x.numel()) * 6)


def layernorm_f32(x, scale, bias, y, m, c, eps=1e-5):
    _launch("layernorm_f32", _p(x), _p(scale), _p(bias), _p(y), int(m), int(c), float(eps), work=float(m) * c * 8)


# ------------------------------------------------------------ image tower --------
def patchify_bf16(img_nhwc, out_bf16, patch):
    _chk(img_nhwc, torch.float32, "img")
    _chk(out_bf16, torch.bfloat16, "out")
    b, s, _, _ = img_nhwc.shape
    _launch("patchify_bf16", _p(img_nhwc), _p(out_bf16), b, s, int(patch), out_bf16.shape[1])


def vit_tokens(patches, class_embedding, position_embedding, out, batch, n_patches, dim):
    _launch("vit_tokens", _p(patches), _p(class_embedding), _p(position_embedding), _p(out), int(batch), int(n_patches),
            int(dim))


def l2norm_rows(x, y):
    _chk(x, torch.float32, "x")
    m, c = x.shape
    _launch("l2norm_rows", _p(x), _p(y), m, c)


# ------------------------------------------------------------ LoRA adapters -------
LORA_RANKS = (4, 8, 16)


def lora_merge(w, down, up, k, n, rank, fwd=None, ldk=0, row_offset=0, dgrad=None, ld_dst=0, col_offset=0, merged=None,
               scale=1.0):
    """bf16(w + scale down @ up) for w fp32 [k, n], down [k, rank], up [rank, n], into the forward operand layout of
    ``prep_weight`` (``fwd``) and / or the dgrad layout of ``prep_weight_dgrad`` (``dgrad``); ``merged``: the fp32 sum"""
    _launch("lora_merge", _p(w), int(k), int(n), _p(down), _p(up), int(rank), float(scale), _p(fwd), int(ldk),
            int(row_offset), _p(dgrad), int(ld_dst), int(col_offset), _p(merged))


def lora_grad(x, dys, downs, ups, d_downs, d_ups, m, k, n, rank, ldx=0, lddy=0, scale=1.0):
    """For adapters i sharing x bf16 [m, k]: d_ups[i] += scale (x downs[i])^T dys[i] and d_downs[i] += scale x^T
    (dys[i] ups[i]^T); dys[i] bf16 [m, n] with row pitch ``lddy``.  One launch reads x and every dy once."""
    g = len(dys)
    assert 1 <= g <= 3 and len(downs) == len(ups) == len(d_downs) == len(d_ups) == g
    need = int(lib().ddpo_lora_grad_workspace_floats(int(rank), g, int(m), int(k), int(n)))
    if need < 0:
        raise ValueError(f"lora_grad: no tiling for k={k}, n={n}, {g} adapters at rank {rank}")
    ws = _workspace("lora_grad", x.device, need)
    arr = lambda ts: (C.c_void_p * g)(*[t.data_ptr() for t in ts])   # noqa: E731
    for t in list(dys) + [x]:
        assert t.is_cuda and t.dtype == torch.bfloat16
    for t in list(downs) + list(ups) + list(d_downs) + list(d_ups):
        assert t.is_cuda and t.dtype == torch.float32
    _launch("lora_grad", _p(x), int(ldx or k), arr(dys), int(lddy or n), arr(downs), arr(ups), arr(d_downs), arr(d_ups),
            g, int(m), int(k), int(n), int(rank), float(scale), _p(ws), ws.numel(), work=float(m) * (k + g * n) * 2,
            tag=f"M{m} K{k} N{n} G{g} r{rank}" if PROFILE is not None else "")
