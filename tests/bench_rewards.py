"""Time per reward call on 8 decoded 512 x 512 images: the reference's host path (PIL / NumPy, as restated in
tests/_rewards_ref.py; CLIP towers on the GPU kernels either way) against the device path of ddpo_b200.training.callbacks,
for each image-symmetry / consistency reward, and the aesthetic reward with its host preprocessing (before) and its
device preprocessing (after).

    python tests/bench_rewards.py [--reps 5] [--out results/bench_rewards.json]

Each figure is the median of --reps calls after one warm-up call, timed with a host clock around a call that ends by
copying its scores to the host (a device synchronise).  The card name and power limit are printed first.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import _rewards_ref as R  # noqa: E402

from ddpo_b200 import clip_vision as CV  # noqa: E402
from ddpo_b200.training import callbacks as C  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = "unknown"
    return f"{name}, power limit / max SM clock: {q}"


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
        del out
    return 1e3 * float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_rewards needs a CUDA device"
    print(card(), flush=True)
    imgs = (np.random.default_rng(0).random((8, 512, 512, 3)) * 255).astype(np.uint8)   # the driver's uint8 hand-off
    prompts = ["a photo of a cat", "a dog", "two horses", "a bird", "a fish", "an owl", "a llama", "a frog"]
    tower = CV.CLIPImageTower(CV.VIT_L14, device="cuda", seed=0)
    consistency = CV.CLIPConsistency(device="cuda", seed=0)

    def feats(t):
        return lambda px: t.image_features(torch.from_numpy(np.ascontiguousarray(px))).cpu().numpy()

    def consistency_host():
        img = consistency.vision.image_features(torch.from_numpy(CV.preprocess(imgs, 224))).cpu().double().numpy()
        txt = consistency.text_features(prompts).cpu().double().numpy()
        return R.consistency(img, txt, np.float32(consistency.logit_scale))

    host = {"mirror": lambda: R.mirror(imgs), "mirror_corr": lambda: R.mirror_corr(imgs),
            "rotational_corr": lambda: R.rotational_corr(imgs),
            "rotational": lambda: R.rotational(imgs, feats(tower), 224),
            "thumbnail": lambda: R.thumbnail(imgs, feats(tower), 224), "consistency": consistency_host}
    rows = []
    for name, h in host.items():
        kw = {"model": consistency} if name == "consistency" else {}
        fn = C.callback_fns[name](**kw)
        dev_ms = timed(lambda: fn(imgs, prompts, {}), args.reps)
        host_ms = timed(h, args.reps)
        rows.append({"reward": name, "host_ms": round(host_ms, 3), "device_ms": round(dev_ms, 3)})
        print(json.dumps(rows[-1]), flush=True)
    sc = CV.AestheticScorer(CV.VIT_L14, device="cuda", seed=0)
    before = timed(lambda: sc.score_features(sc.image_features(torch.from_numpy(CV.preprocess(imgs, 224)))).cpu(),
                   args.reps)
    after = timed(lambda: sc(imgs), args.reps)
    rows.append({"reward": "aesthetic", "host_ms": round(before, 3), "device_ms": round(after, 3)})
    print(json.dumps(rows[-1]), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"card": card(), "images": "8 x 512 x 512 uint8", "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
