"""Harness shared by the layer-by-layer gradient tests (test_backward_layers.py, test_param_grad_layers.py): the backend a
check runs on (the CUDA library or its torch-CPU emulation), guarded output buffers whose outside must come back
unchanged, the error bounds and the checks that apply them.  Every check stores its measured errors as test
properties (``pytest --junitxml=...`` writes them out), so that the margins of the bounds are on record."""
import pytest
import torch

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64

# Bounds.  The worst errors of the CUDA kernels over all cases of test_backward_layers.py, measured on an H100 80GB HBM3
# (700 W), are in the comments.  The fp32, bf16-L2 and attention-L2 bounds are the rest of the suite's, not fitted to
# these numbers.
F32_MAX, F32_L2 = 2e-3, 1e-3          # fp32 outputs (fp32 accumulation of bf16 operands): worst 1.6e-5, 1.3e-5
BF16_MAX, BF16_L2 = 8e-3, 4e-3        # bf16 outputs, whose rounding alone is up to 2^-8 of the value: worst 3.5e-3, 1.7e-3
ATT_MAX, ATT_L2 = 2e-2, 2e-2          # attention gradients (P and dS pass through bf16): worst 4.7e-3, 2.8e-3
SUM_TOL = 1e-5                        # reductions, in units of sum |term|: worst 0.33 of the bound (dense_small dW)
F32_ULP = 2.0 ** -23                  # one fp32 rounding of an accumulate-into (out = old + sum)
# test_forward_layers.py, same H100.  Timestep sin/cos: |err| <= SINCOS_ARG_ULPS ulp of the argument t * freq (fp32
# rounding of freq and of the product) + SINCOS_ULPS ulp: worst 0.63 of the bound.  Norms of inputs at a DC offset of
# up to 64 sigma: no worse than NORM_DC_FACTOR x the error of torch fp32 with var = E[x^2] - E[x]^2 (or the standard
# bound, if larger): worst 2.2 x torch (GroupNorm two-pass y_f32, 64 sigma), which is still inside F32_MAX.
SINCOS_ARG_ULPS, SINCOS_ULPS = 3, 4
NORM_DC_FACTOR = 4


class Backend:
    """The ops module a check runs on: the CUDA library, or its torch-CPU emulation."""

    def __init__(self, name):
        self.emulated = name == "emulator"
        if self.emulated:
            import _cpu_ops_emulator as ops
            self.dev = "cpu"
        else:
            from ddpo_b200 import ops
            self.dev = "cuda"
        self.ops = ops
        # extra columns past the pitch for ops that take a row pitch; the emulator writes dense outputs (it has no
        # ld_out), so its outputs get extra rows only
        self.pad = 0 if self.emulated else 64

    def sync(self):
        if not self.emulated:
            torch.cuda.synchronize()


def _backend_params(small, large=()):
    """(backend, *case) parameter sets: small cases on both backends, large ones on the GPU only"""
    out = []
    for case in small:
        out.append(pytest.param("emulator", *case, id="emu-" + "-".join(map(str, case))))
    for case in list(small) + list(large):
        out.append(pytest.param("cuda", *case, marks=pytest.mark.gpu, id="cuda-" + "-".join(map(str, case))))
    return out


_NODE = {}


@pytest.fixture(autouse=True)
def _current_node(request):
    """the running test, for _record (a test module activates this fixture by importing it)"""
    _NODE["node"] = request.node
    yield
    _NODE.pop("node", None)


def _record(name, **vals):
    node = _NODE.get("node")
    if node is not None:
        node.user_properties.append((name, " ".join(f"{k}={v:.3g}" if isinstance(v, float) else f"{k}={v}"
                                                    for k, v in vals.items())))


class Guarded:
    """A [rows, cols] output at the top-left of a larger buffer: ``extra_cols`` past the pitch, ``extra_rows`` after the
    last row.  The buffer starts as seeded noise (``init`` goes into the view) and everything outside the view must
    come back unchanged (``check``)."""

    def __init__(self, rows, cols, dtype, dev, extra_cols=0, extra_rows=8, init=None, seed=99):
        g = torch.Generator().manual_seed(seed)
        self.buf = (torch.randn(rows + extra_rows, cols + extra_cols, generator=g) * 1e3 + 4097.0).to(dtype).to(dev)
        self.rows, self.cols, self.ld = rows, cols, cols + extra_cols
        if init is not None:
            self.view.copy_(init.reshape(rows, cols))
        self.snapshot = self.buf.clone()

    @property
    def view(self):
        return self.buf[:self.rows, :self.cols]

    @property
    def arg(self):
        """what to hand to an op: the dense view where there are no extra columns, else the whole pitched buffer"""
        return self.view if self.ld == self.cols else self.buf

    def check(self, what):
        outside = torch.ones(self.buf.shape, dtype=torch.bool, device=self.buf.device)
        outside[:self.rows, :self.cols] = False
        assert torch.equal(self.buf[outside], self.snapshot[outside]), f"{what}: write outside the output"


class FlatSlot:
    """A parameter-gradient slot the way ``UNet.g(name)`` hands it out: a dense [rows, cols] fp32 view at a 64-float
    (256-byte) aligned offset inside a 1-D buffer.  The slot starts from ``init`` (a non-zero prior gradient: the
    train pass always accumulates), the rest of the buffer (the neighbouring parameters) is seeded noise that must come
    back bit-identical (``check``).  ``before`` and ``after`` are the float counts of the neighbours, rounded up to a
    multiple of 64."""

    def __init__(self, rows, cols, dev, init, before=64, after=256, seed=98):
        before, after = -(-before // 64) * 64, -(-after // 64) * 64
        n = rows * cols
        g = torch.Generator().manual_seed(seed)
        self.buf = (torch.randn(before + n + after, generator=g) * 1e3 + 4097.0).to(dev)
        self.off, self.n, self.shape = before, n, (rows, cols)
        self.view.copy_(init.reshape(rows, cols))
        self.snapshot = self.buf.clone()

    @property
    def view(self):
        return self.buf[self.off:self.off + self.n].view(self.shape)

    def prior(self):
        return self.snapshot[self.off:self.off + self.n].view(self.shape)

    def check(self, what):
        assert torch.equal(self.buf[:self.off], self.snapshot[:self.off]), f"{what}: write before the slot"
        assert torch.equal(self.buf[self.off + self.n:], self.snapshot[self.off + self.n:]), f"{what}: write after the slot"


def check_close(name, out, ref, max_tol, l2_tol):
    d = out.double() - ref
    rmax = ref.abs().max().item()
    e_max = d.abs().max().item() / rmax
    e_l2 = (d.norm() / ref.norm()).item()
    _record(name, max=e_max, l2=e_l2)
    assert e_max <= max_tol and e_l2 <= l2_tol, \
        f"{name}: max err {e_max:.3g} * max|ref| (bound {max_tol}), relative L2 {e_l2:.3g} (bound {l2_tol})"


def check_sum(name, out, ref, abs_terms, tol=SUM_TOL, old=None):
    """out (+)= a sum: |out - old - ref| <= tol * sum|terms| (+ one rounding of the add into ``old``)"""
    o = out.double()
    err = (o - (old.double() if old is not None else 0) - ref).abs()
    bound = tol * abs_terms + (2 * F32_ULP * o.abs() if old is not None else 0) + 1e-30
    worst = (err / bound).max().item()
    _record(name, worst_over_bound=worst, rel_to_abs_sum=(err / (abs_terms + 1e-30)).max().item())
    assert worst <= 1.0, f"{name}: error {worst:.3g} x the bound ({tol} * sum|terms|)"


def rnd(g, *shape, scale=1.0, shift=0.0):
    return torch.randn(*shape, generator=g) * scale + shift
