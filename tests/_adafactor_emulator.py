"""TEST INFRASTRUCTURE: torch-CPU emulation of ``ops.adafactor_plan`` / ``ops.clip_adafactor`` for the host dry runs
(tests/_cpu_ops_emulator.py covers the other ops): the real host planner, and the arithmetic of the NumPy restatement
tests/_adafactor_ref.py on its factoring decisions.  ``install(E)`` adds both to an emulator module."""
import numpy as np
import torch

from ddpo_b200 import ops as _real_ops

import _adafactor_ref as A  # noqa: E402

adafactor_plan = _real_ops.adafactor_plan


def clip_adafactor(params, grad_acc, state, plan, workspace, sumsq, grad_scale, max_norm, lr, wd, step, norm_out=None):
    """the oracle's arithmetic (tests/_adafactor_ref.py) on the tensors and factoring decisions of the real planner"""
    lr, wd = float(np.float32(lr)), float(np.float32(wd))
    norm = float(np.float32(grad_scale) * np.sqrt(np.float32(sumsq.item())))
    g = grad_acc.numpy() * np.float32(grad_scale)
    if not norm < max_norm:
        g = (g / np.float32(norm)) * np.float32(max_norm)
    beta = A.beta_t(int(step) - 1)
    p = params.numpy()
    for t, (views, shape) in enumerate(zip(plan.state_views(state), plan.shapes)):
        off, n, kind = int(plan.tensors[t][0]), int(np.prod(shape)), plan.kinds[t]
        fd = None if kind == 0 else ((len(shape) - 2, len(shape) - 1) if kind == 1 else (len(shape) - 1, len(shape) - 2))
        leaf = {k: v.numpy().copy() for k, v in views.items()}
        u = A.scale_by_factored_rms(g[off:off + n].reshape(shape), leaf, beta, fd)
        new, denom, pscale = A.tensor_update(p[off:off + n].reshape(shape), u, lr, wd)
        p[off:off + n] = new.reshape(-1)
        for k, v in views.items():
            v.copy_(torch.from_numpy(leaf[k]))
        workspace[2 * t], workspace[2 * t + 1] = float(denom), float(pscale)
    grad_acc.zero_()
    if norm_out is not None:
        norm_out.fill_(norm)


def install(emulator):
    emulator.adafactor_plan, emulator.clip_adafactor = adafactor_plan, clip_adafactor
