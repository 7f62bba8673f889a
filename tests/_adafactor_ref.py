"""TEST INFRASTRUCTURE: NumPy restatement of the reference's Adafactor chain
``optax.chain(clip_by_global_norm(max_grad_norm), adafactor(learning_rate=lr, weight_decay_rate=wd))``
(reference ``pipeline/policy_gradient.py:132-150``; optax==0.1.5 with every other adafactor argument at its default:
min_dim_size_to_factor 128, decay_rate 0.8, decay_offset 0, multiply_by_parameter_scale, clipping_threshold 1,
momentum None, eps 1e-30, factored) over the ``(offset, shape)`` views of the flat buffer, in float32 or float64, and
of ``AccumulatingTrainState.apply_gradients`` with it."""
import numpy as np

f32 = np.float32


def factored_dims(shape, min_dim_size_to_factor=128):
    """optax ``_factored_dims``: None, or (d1, d0) = the last two entries of argsort(shape)."""
    if len(shape) < 2:
        return None
    sd = np.argsort(shape)
    if shape[sd[-2]] < min_dim_size_to_factor:
        return None
    return int(sd[-2]), int(sd[-1])


class AdafactorState:
    def __init__(self, tensors, dtype=f32, min_dim_size_to_factor=128):
        self.count = 0
        self.min_dim = min_dim_size_to_factor
        self.leaves = []
        for _, shape in tensors:
            fd = factored_dims(shape, min_dim_size_to_factor)
            if fd is None:
                self.leaves.append({"v": np.zeros(shape, dtype)})
            else:
                d1, d0 = fd
                self.leaves.append({"v_row": np.zeros(np.delete(shape, d0), dtype),
                                    "v_col": np.zeros(np.delete(shape, d1), dtype)})


def scale_by_factored_rms(g, leaf, beta, fd):
    """``fd``: factored_dims(g.shape) or None.  Updates ``leaf`` in place, returns u."""
    dt = g.dtype.type
    G = g * g + dt(1e-30)
    if fd is None:
        leaf["v"] = (dt(beta) * leaf["v"] + dt(1 - beta) * G).astype(dt)
        return g * leaf["v"] ** dt(-0.5)
    d1, d0 = fd
    leaf["v_row"] = (dt(beta) * leaf["v_row"] + dt(1 - beta) * G.mean(axis=d0)).astype(dt)
    leaf["v_col"] = (dt(beta) * leaf["v_col"] + dt(1 - beta) * G.mean(axis=d1)).astype(dt)
    rcm = leaf["v_row"].mean(axis=d1 - 1 if d1 > d0 else d1, keepdims=True)
    row_factor = (leaf["v_row"] / rcm) ** dt(-0.5)
    col_factor = leaf["v_col"] ** dt(-0.5)
    return g * np.expand_dims(row_factor, d0) * np.expand_dims(col_factor, d1)


def tensor_update(p, u, lr, wd):
    """clip_by_block_rms(1) -> scale(lr) -> scale_by_param_block_rms -> add_decayed_weights(wd) -> scale(-1), applied.
    Returns (p_new, clip denominator, param scale)."""
    dt = p.dtype.type
    denom = np.maximum(dt(1), np.sqrt(np.mean(u * u)))
    u = u / denom
    u = u * dt(lr)
    pscale = np.sqrt(np.maximum(np.mean(p * p), dt(1e-6)))
    u = u * pscale
    u = u + dt(wd) * p
    return (p - u).astype(dt), dt(denom), dt(pscale)


def beta_t(count, dtype=f32):
    """optax _decay_rate_pow at the number of earlier updates: 1 - (count + 1)^-0.8 (optax forms it in float32)"""
    return 1.0 - float(dtype(count + 1) ** dtype(-0.8))


def clip_adafactor_update(params, grads, tensors, st, lr=1e-5, wd=1e-4, max_norm=1.0, dtype=f32):
    """One update of the flat buffer; padding floats between tensors are returned unchanged.
    Returns (params, global norm, [(denom, pscale)] per tensor)."""
    p = np.asarray(params, dtype).copy()
    g = np.asarray(grads, dtype)
    gn = np.sqrt(np.sum(np.asarray(g, np.float64) ** 2)).astype(dtype)
    if not (gn < dtype(max_norm)):
        g = ((g / gn) * dtype(max_norm)).astype(dtype)
    beta = beta_t(st.count, dtype)
    stats = []
    for (off, shape), leaf in zip(tensors, st.leaves):
        n = int(np.prod(shape))
        pt, gt = p[off:off + n].reshape(shape), g[off:off + n].reshape(shape)
        u = scale_by_factored_rms(gt, leaf, beta, factored_dims(shape, st.min_dim))
        new, denom, pscale = tensor_update(pt, u, lr, wd)
        p[off:off + n] = new.reshape(-1)
        stats.append((denom, pscale))
    st.count += 1
    return p, gn, stats


class AccumulatingTrainState:
    """grad_acc += g; on do_update: g~ = (grad_acc + g)/(n_acc+1) -> clip + adafactor -> zero."""

    def __init__(self, params, tensors, dtype=f32, **hp):
        self.params = np.asarray(params, dtype).copy()
        self.tensors = list(tensors)
        self.grad_acc = np.zeros_like(self.params)
        self.n_acc = 0
        self.step = 0
        self.opt = AdafactorState(self.tensors, dtype)
        self.hp = hp
        self.dtype = dtype

    def apply_gradients(self, grads, do_update):
        g = np.asarray(grads, self.dtype)
        if do_update:
            gm = ((self.grad_acc + g) / self.dtype(self.n_acc + 1)).astype(self.dtype)
            self.params, gn, _ = clip_adafactor_update(self.params, gm, self.tensors, self.opt, dtype=self.dtype, **self.hp)
            self.grad_acc[:] = 0
            self.n_acc = 0
            self.step += 1
            return gn
        self.grad_acc = (self.grad_acc + g).astype(self.dtype)
        self.n_acc += 1
        return None
