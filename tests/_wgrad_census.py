"""Every weight-gradient GEMM (``ops.wgrad``) of one PPO train pass, ``UNet.backward`` at batch 40, for SD2-base, SD1
and the TINY / SMALL widths, recorded on the ``meta`` device the way tests/_igemm_census.py records the implicit GEMM.
Used by test_wgrad_plan_cpu.py and bench_wgrad_plan.py."""
import functools

import torch

import _forward_census as census_mod
import _igemm_census as ic
from ddpo_b200 import unet as unet_mod
from ddpo_b200 import unet_spec

BATCH = 40
CONFIGS = {"sd2": unet_spec.SD2_BASE, "sd1": unet_spec.SD1, "tiny": unet_spec.TINY, "small": unet_spec.SMALL}


@functools.lru_cache(maxsize=None)
def calls(cfg_name):
    """the wgrad ``Call``s of one train pass, in launch order"""
    cfg = CONFIGS[cfg_name]
    rec = ic._Recorder()
    saved = unet_mod.ops
    unet_mod.ops = rec
    try:
        _, total = unet_spec.param_offsets(cfg)
        net = unet_mod.UNet(cfg, torch.empty(total, device="meta"), device="meta")
        net.enable_training()
        rec.params = net.params if net.params._base is None else net.params._base
        rec.batch, rec.recording = BATCH, True
        net.prepare_context(torch.empty(BATCH, cfg.ctx_len, cfg.cross_attention_dim, device="meta"))
        s = cfg.sample_size
        lat = torch.empty(BATCH, cfg.in_channels, s, s, device="meta")
        tape = []
        net.forward(lat, torch.empty(BATCH, dtype=torch.int32, device="meta"), tape=tape)
        net.backward(tape, torch.empty_like(lat))
    finally:
        unet_mod.ops = saved
    return [c for c in rec.calls if c.op == "wgrad"]


def shape(call):
    """(m, c0, c1, n, taps) of a wgrad call: m counts the pixels of dY"""
    a = call.args
    m = a["conv"][0] * a["conv"][1] * a["conv"][2] if a.get("conv") else a["m"]
    return m, a["c0"], a.get("c1", 0), a["n"], a.get("taps", 1)


def distinct(cfg_name):
    """[(Call, number of calls)] per distinct signature, in first-call order"""
    return [(c, n) for _, c, n in census_mod._distinct(calls(cfg_name))]


def old_plan(m, c0, c1, n, taps, sms=132):
    """(splits, [CTAs of each launch]) of the planner this one replaced: 128-channel blocks per (tap, source), a
    256-wide launch and a launch for the 64 / 128 / 192-column remainder, and pixel splits for ~2 waves of both"""
    pb = -(-m // 64)
    mt = taps * (-(-c0 // 128) + -(-c1 // 128))
    widths = [256] * (n // 256) + ([n % 256] if n % 256 else [])
    s = -(-2 * sms // (mt * len(widths)))
    s = max(1, min(s, pb // 8))
    while s > 1 and taps * (c0 + c1) * n * s > 48 << 20:
        s -= 1
    launches = [mt * s * (n // 256)] if n >= 256 else []
    if n % 256:
        launches.append(mt * s)
    return s, launches
