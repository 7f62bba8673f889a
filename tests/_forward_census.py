"""The U-Net forward's and the VAE's kernel launches, recorded without a GPU: ``UNet.prepare_context`` and
``UNet.forward``, ``VAEDecoder.decode`` and ``VAEEncoder.encode`` run on the ``meta`` device with the model module's
``ops`` swapped for a recorder, so every launch's arguments (scalars, and the shape, dtype, strides and storage offset
of every tensor) are listed exactly as unet.py / vae.py make them.  test_forward_layers.py and test_vae_layers.py replay
each distinct configuration on the CUDA library against float64.

A launch's *signature* is its op name and its arguments with every tensor reduced to (shape, dtype, strides, buffer,
offset): ``buffer`` numbers the distinct storages of the call in order of first use ("P" for the flat parameter buffer,
whose offsets are the parameters' and vary by layer), ``offset`` is the tensor's element offset from the first tensor of
the call on the same storage.  So q/k/v column slices of one ``qkv`` buffer keep their relation, and two layers that
differ only in which parameters they read share a signature."""
import functools
import hashlib
import inspect

import torch

from ddpo_b200 import ops as real_ops
from ddpo_b200 import unet as unet_mod
from ddpo_b200 import unet_spec
from ddpo_b200 import vae as vae_mod

# (name, config, batch, taped): sampling runs the U-Net at batch 2 x 8 (CFG), the PPO train pass at 40 with a tape
RUNS = [("sd2", unet_spec.SD2_BASE, 16, False), ("sd2", unet_spec.SD2_BASE, 40, True),
        ("sd1", unet_spec.SD1, 16, False), ("sd1", unet_spec.SD1, 40, True)]
TINY_RUNS = [("tiny", unet_spec.TINY, 2, False), ("tiny", unet_spec.TINY, 3, True)]
# (part, config, chunk batch): the VAE runs ``decode_batch`` = 2 images per chunk (a sampling batch of 8 is four
# chunks), and a batch of odd size ends with a chunk of 1
VAE_RUNS = [("decoder", vae_mod.SD_VAE, 2), ("decoder", vae_mod.SD_VAE, 1),
            ("encoder", vae_mod.SD_VAE, 2), ("encoder", vae_mod.SD_VAE, 1)]
VAE_MICRO_RUNS = [("decoder", vae_mod.VAE_MICRO, 2), ("decoder", vae_mod.VAE_MICRO, 1),
                  ("encoder", vae_mod.VAE_MICRO, 2), ("encoder", vae_mod.VAE_MICRO, 1)]

PASS_THROUGH = ("gn_stats_shape", "groupnorm_workspace_floats")


class Tensor:
    """what a replay needs of one tensor argument"""
    __slots__ = ("shape", "dtype", "stride", "buf", "offset")

    def __init__(self, shape, dtype, stride, buf, offset):
        self.shape, self.dtype, self.stride, self.buf, self.offset = shape, dtype, stride, buf, offset

    def key(self):
        return ("T", self.shape, str(self.dtype), self.stride, self.buf, self.offset)

    def __repr__(self):
        return f"T{list(self.shape)}{str(self.dtype)[6:]}@{self.buf}+{self.offset}"


class Call:
    """one launch: ``args`` maps the op's parameter names to scalars, ``Tensor``s or None; ``batch`` is the number of
    samples the launch covers (the U-Net batch, the VAE chunk, 1 inside the VAE attention's per-sample loop),
    ``group_table`` the (w_off, b_off, y_off, n) entries of a dense_small_grouped launch, ``role`` what a VAE attention
    GEMM computes ("vt": V^T = Wv^T g^T, "qk": Q K^T, "pv": P V), whose operands are not a weight and activations"""

    def __init__(self, op, args, batch, group_table=None, role=None):
        self.op, self.args, self.batch, self.group_table, self.role = op, args, batch, group_table, role

    def key(self):
        items = tuple((k, v.key() if isinstance(v, Tensor) else v) for k, v in sorted(self.args.items()))
        key = (self.op, items, tuple(self.group_table) if self.group_table else None)
        return key + (self.role,) if self.role else key

    def tag(self):
        """a short readable name of the configuration (test ids)"""
        a = self.args
        t = lambda k: a.get(k) if isinstance(a.get(k), Tensor) else None
        if self.op == "igemm":
            rows = a["conv"][0] * a["conv"][1] * a["conv"][2] if a.get("conv") else a["m"]
            k = a.get("taps", 1) * a["c0"]
            flags = [f for f in ("bias", "rowvec", "residual", "out_f32", "out_bf16", "aux_bf16", "gn_stats")
                     if t(f) is not None]
            kind = f"conv{a.get('taps', 1)}s{a.get('stride', 1)}" if a.get("conv") else "lin"
            kind = self.role or kind + ("-nolowpad" if a.get("no_low_pad") else "")
            return f"{kind}-M{rows}-N{a['n']}-K{k}" + ("-geglu" if a.get("geglu") else "") + "-" + "+".join(flags)
        if self.op == "attention_fwd":
            hd = a.get("head_dim", 64)
            return f"B{a['batch']}-H{a['heads']}-d{hd}-nq{a['nq']}-nk{a['nk']}" + ("-lse" if t("lse") else "")
        if self.op == "groupnorm_fwd":
            outs = "+".join(f for f in ("y_bf16", "y_f32", "raw_bf16", "stats0") if t(f) is not None)
            eps = f"-eps{a['eps']:g}" if "eps" in a else ""
            return f"B{a['batch']}-hw{a['hw']}-c{a['c0']}+{a.get('c1', 0)}-silu{int(a.get('silu', True))}{eps}-{outs}"
        if self.op == "layernorm_fwd":
            return f"m{a['m']}-c{a['c']}"
        first = next(v for v in a.values() if isinstance(v, Tensor))
        dims = [str(v) for k, v in sorted(a.items()) if isinstance(v, int) and not isinstance(v, bool)]
        return f"B{self.batch}-" + "x".join(map(str, first.shape)) + "".join("-" + d for d in dims)

    def test_id(self):
        """the configuration's test id: readable tag plus a digest of the whole signature"""
        return f"{self.op}-{self.tag()}-{hashlib.sha1(repr(self.key()).encode()).hexdigest()[:6]}"


class _Recorder:
    """stands in for the ``ops`` module: pure helpers pass through, every other attribute records its calls"""

    def __init__(self):
        self.calls = []
        self.recording = False
        self.params = None
        self.weights = None      # ids of a VAE's prepared GEMM weights: tells the attention's per-sample GEMMs apart
        self._tables = {}

    def dense_small_group_table(self, entries, device):
        tab, ctas = real_ops.dense_small_group_table(entries, "cpu")
        t = torch.empty(tab.shape, dtype=tab.dtype, device=device)
        self._tables[id(t)] = (t, [tuple(int(v) for v in e) for e in entries])
        return t, ctas

    def __getattr__(self, name):
        if name in PASS_THROUGH:
            return getattr(real_ops, name)
        sig = inspect.signature(getattr(real_ops, name))

        def record(*args, **kwargs):
            if not self.recording:
                return None
            bound = sig.bind(*args, **kwargs).arguments
            bases, firsts, out = {}, {}, {}
            table = None
            for k, v in bound.items():
                if v is None or (not isinstance(v, torch.Tensor) and v == sig.parameters[k].default):
                    continue     # an argument passed at its default is the same launch as one left out
                if not isinstance(v, torch.Tensor):
                    out[k] = v
                    continue
                if id(v) in self._tables:
                    table = self._tables[id(v)][1]
                base = v._base if v._base is not None else v
                if base is self.params:
                    buf, off = "P", 0
                else:
                    buf = bases.setdefault(id(base), len(bases))
                    off = v.storage_offset() - firsts.setdefault(buf, v.storage_offset())
                out[k] = Tensor(tuple(v.shape), v.dtype, tuple(v.stride()), buf, off)
            role, batch = self._vae_role(name, bound)
            self.calls.append(Call(name, out, batch, table, role))
        return record

    def _vae_role(self, name, bound):
        """(role, samples covered): the VAE attention runs its score GEMMs and softmax once per sample, whatever the
        chunk batch"""
        if self.weights is None:
            return None, self.batch
        if name == "softmax_rows":
            return None, 1
        if name == "igemm":
            if id(bound["a0"]) in self.weights:
                return "vt", 1
            if id(bound["wt"]) not in self.weights:
                return ("qk" if bound.get("out_f32") is not None else "pv"), 1
        return None, self.batch


def _record_run(cfg, batch, taped):
    rec = _Recorder()
    saved = unet_mod.ops
    unet_mod.ops = rec
    try:
        _, total = unet_spec.param_offsets(cfg)
        net = unet_mod.UNet(cfg, torch.empty(total, device="meta"), device="meta")
        rec.params = net.params if net.params._base is None else net.params._base
        rec.batch, rec.recording = batch, True
        ctx = torch.empty(batch, cfg.ctx_len, cfg.cross_attention_dim, device="meta")
        net.prepare_context(ctx)
        n_ctx = len(rec.calls)
        s = cfg.sample_size
        lat = torch.empty(batch, cfg.in_channels, s, s, device="meta")
        ts = torch.empty(batch, dtype=torch.int32, device="meta")
        net.forward(lat, ts, tape=[] if taped else None)
    finally:
        unet_mod.ops = saved
    return rec.calls[:n_ctx], rec.calls[n_ctx:]


@functools.lru_cache(maxsize=None)
def runs(which="full"):
    """{(model, batch, taped): (prepare_context calls, forward calls)}"""
    return {(name, b, taped): _record_run(cfg, b, taped) for name, cfg, b, taped in (RUNS if which == "full" else TINY_RUNS)}


def _distinct(calls):
    """[(signature key, Call, number of launches)] in first-launch order; launches that share a signature cover the same
    number of samples"""
    seen = {}
    for c in calls:
        k = c.key()
        if k in seen:
            assert seen[k][1].batch == c.batch, (c.test_id(), seen[k][1].batch, c.batch)
            seen[k][2] += 1
        else:
            seen[k] = [k, c, 1]
    return [tuple(v) for v in seen.values()]


@functools.lru_cache(maxsize=None)
def census(which="full"):
    """the distinct configurations, in first-launch order: [(signature key, Call, number of launches)]"""
    return _distinct(c for ctx_calls, fwd_calls in runs(which).values() for c in ctx_calls + fwd_calls)


def _record_vae_run(part, cfg, batch):
    rec = _Recorder()
    saved = vae_mod.ops
    vae_mod.ops = rec
    try:
        cls = vae_mod.VAEDecoder if part == "decoder" else vae_mod.VAEEncoder
        _, total = vae_mod.param_offsets(cfg, part=part)
        net = cls(cfg, torch.empty(total, device="meta"), device="meta", decode_batch=batch)
        rec.params = net.params if net.params._base is None else net.params._base
        rec.weights = {id(t) for t in net.w.values()}
        rec.batch, rec.recording = batch, True
        s = cfg.sample_size
        up = 2 ** (len(cfg.block_out_channels) - 1)
        if part == "decoder":
            net.decode(torch.empty(batch, cfg.latent_channels, s, s, device="meta"))
        else:
            net.encode(torch.empty(batch, s * up, s * up, cfg.out_channels, device="meta"))
    finally:
        vae_mod.ops = saved
    return rec.calls


@functools.lru_cache(maxsize=None)
def vae_runs(which="full"):
    """{(part, chunk batch): the launches of one chunk}"""
    return {(part, b): _record_vae_run(part, cfg, b)
            for part, cfg, b in (VAE_RUNS if which == "full" else VAE_MICRO_RUNS)}


@functools.lru_cache(maxsize=None)
def vae_census(which="full"):
    """the VAE's distinct configurations (``census`` of the decoder and encoder runs)"""
    return _distinct(c for calls in vae_runs(which).values() for c in calls)
