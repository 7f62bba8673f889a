"""Every implicit-GEMM launch of one SD2-base denoising step (the U-Net at batch 2 x 8 with CFG) and of one PPO train
pass (forward with a tape and ``UNet.backward`` at batch 40), recorded on the ``meta`` device the way
tests/_forward_census.py records the forward.  Used by test_igemm_plan_cpu.py and bench_igemm_plan.py."""
import functools

import torch

import _forward_census as census_mod
from ddpo_b200 import unet as unet_mod
from ddpo_b200 import unet_spec

PASSES = {"sample": (16, False), "train": (40, True)}


class _Recorder(census_mod._Recorder):
    """the forward census's recorder, also passing through the workspace-size helpers the backward calls"""

    def __getattr__(self, name):
        if name.endswith("_workspace_floats"):
            return getattr(census_mod.real_ops, name)
        return super().__getattr__(name)


@functools.lru_cache(maxsize=None)
def launches(pass_name, cfg=unet_spec.SD2_BASE):
    """the igemm ``Call``s of one pass, in launch order"""
    batch, train = PASSES[pass_name]
    rec = _Recorder()
    saved = unet_mod.ops
    unet_mod.ops = rec
    try:
        _, total = unet_spec.param_offsets(cfg)
        net = unet_mod.UNet(cfg, torch.empty(total, device="meta"), device="meta")
        if train:
            net.enable_training()
        rec.params = net.params if net.params._base is None else net.params._base
        rec.batch, rec.recording = batch, True
        net.prepare_context(torch.empty(batch, cfg.ctx_len, cfg.cross_attention_dim, device="meta"))
        s = cfg.sample_size
        lat = torch.empty(batch, cfg.in_channels, s, s, device="meta")
        tape = [] if train else None
        net.forward(lat, torch.empty(batch, dtype=torch.int32, device="meta"), tape=tape)
        if train:
            net.backward(tape, torch.empty_like(lat))
    finally:
        unet_mod.ops = saved
    return [c for c in rec.calls if c.op == "igemm"]


def shape(call):
    """(M, N, K, geglu) of an igemm launch"""
    a = call.args
    m = a["conv"][0] * a["conv"][1] * a["conv"][2] if a.get("conv") else a["m"]
    return m, a["n"], a.get("taps", 1) * (a["c0"] + a.get("c1", 0)), bool(a.get("geglu"))


def distinct(pass_name):
    """[(Call, number of launches)] per distinct signature, in first-launch order"""
    return [(c, n) for _, c, n in census_mod._distinct(launches(pass_name))]


def old_width(n, geglu=False):
    """the tile width the library chose from N alone, with 128-row tiles, before tiles were planned per shape"""
    for w in ((256, 192, 128, 64) if geglu else (128, 160, 192, 96, 64, 32)):
        if n % w == 0:
            return w
