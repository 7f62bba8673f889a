"""CPU tests: the C-ABI library loads and exports every symbol the header declares (no compute calls without
a GPU), header <-> ctypes agreement, host-side logic (PRNG key lineage, stat tracker, parser, prompts, rewards)."""
import ctypes
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_functions():
    src = open(os.path.join(ROOT, "include", "ddpo_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(ddpo_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from ddpo_b200 import _lib, build
    if not os.path.exists(_lib.LIB_PATH):
        build.build()
    L = ctypes.CDLL(_lib.LIB_PATH)
    fns = _header_functions()
    assert len(fns) >= 40
    for f in fns:
        assert hasattr(L, f), f"{f} declared in include/ddpo_b200.h but not exported"
    assert sorted(_lib.SIGNATURES) == fns, set(fns) ^ set(_lib.SIGNATURES)
    lib = _lib.lib()
    assert lib.ddpo_abi_version() == 3


def test_no_gpu_calls_fail_loudly():
    import torch
    if torch.cuda.is_available():
        return
    from ddpo_b200 import _lib
    n = _lib.lib().ddpo_device_sm_count()
    assert n < 0 and b"CUDA" in _lib.lib().ddpo_last_error()
    import pytest
    from ddpo_b200 import ops
    with pytest.raises(AssertionError):
        ops.cast_bf16(torch.zeros(8), torch.zeros(8, dtype=torch.bfloat16))  # CPU tensors are rejected, no fallback


def test_struct_layouts_match_header_order():
    """field order of the ctypes structures == declaration order in the header"""
    from ddpo_b200 import _lib
    src = open(os.path.join(ROOT, "include", "ddpo_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    for cname, st in (("ddpo_ddim_common", _lib.DdimCommon), ("ddpo_igemm_args", _lib.IGemmArgs),
                      ("ddpo_groupnorm_args", _lib.GroupNormArgs), ("ddpo_attention_args", _lib.AttentionArgs),
                      ("ddpo_wgrad_args", _lib.WgradArgs), ("ddpo_attention_bwd_args", _lib.AttentionBwdArgs)):
        body = re.search(r"typedef struct \{([^{}]*)\}\s*" + cname + ";", src, flags=re.S).group(1)
        names = []
        for decl in body.split(";"):
            decl = decl.strip()
            if not decl:
                continue
            for part in decl.split(","):
                found = re.findall(r"([A-Za-z_][A-Za-z0-9_]*)\s*$", part.strip())
                if found:
                    names.append(found[0])
        assert names == [f[0] for f in st._fields_], (cname, names, [f[0] for f in st._fields_])


def test_ctypes_prototypes_match_the_header():
    """every prototype in include/ddpo_b200.h against the ctypes table: parameter count, and per parameter pointer-vs-scalar
    and integer-vs-float class (a drifted signature corrupts the call silently)"""
    from ddpo_b200 import _lib
    src = open(os.path.join(ROOT, "include", "ddpo_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    protos = re.findall(r"\b[A-Za-z_][A-Za-z0-9_ ]*[ *]+(ddpo_[a-z0-9_]+)\s*\(([^()]*)\)\s*;", src)
    assert len(protos) >= 40
    seen = set()
    for name, params in protos:
        seen.add(name)
        params = [q.strip() for q in params.split(",")] if params.strip() not in ("", "void") else []
        restype, argtypes = _lib.SIGNATURES[name]
        assert len(params) == len(argtypes), (name, params, argtypes)
        for q, t in zip(params, argtypes):
            is_ptr_c = "*" in q or "[" in q   # array parameters decay to pointers
            is_ptr_py = t in (ctypes.c_void_p, ctypes.c_char_p) or hasattr(t, "contents") or getattr(t, "_type_", None) == "P"
            assert is_ptr_c == is_ptr_py, (name, q, t)
            if not is_ptr_c:
                is_float_c = bool(re.match(r"(const\s+)?(float|double)\b", q))
                is_float_py = t in (ctypes.c_float, ctypes.c_double)
                assert is_float_c == is_float_py, (name, q, t)
                if re.match(r"(const\s+)?(long long|int64_t|unsigned long long|uint64_t|size_t)\b", q):
                    assert ctypes.sizeof(t) == 8, (name, q, t)
    assert seen == set(_lib.SIGNATURES)


def test_host_threefry_matches_oracle_lineage():
    from ddpo_b200 import ops
    from oracle import threefry as T
    key = ops.prng_key(42)
    assert list(key) == T.PRNGKey(42).tolist()
    a = ops.threefry_split(key, 2)
    assert [list(k) for k in a] == T.split(T.PRNGKey(42)).tolist()
    b = ops.threefry_split(a[1], 8)
    assert [list(k) for k in b] == T.split(np.array(a[1], np.uint32), 8).tolist()


def test_stat_tracker_and_global_advantages():
    from ddpo_b200.utils.stat_tracking import PerPromptStatTracker, global_advantages
    tr = PerPromptStatTracker(4, 2)
    prompts = np.array(["a", "a", "b"])
    r = np.array([1.0, 3.0, 10.0])
    adv = tr.update(prompts, r)
    np.testing.assert_allclose(adv[:2], (r[:2] - 2.0) / (1.0 + 1e-6))           # own stats (count 2 >= min_count)
    np.testing.assert_allclose(adv[2], (10.0 - r.mean()) / (r.std() + 1e-6))      # batch stats (count 1 < 2)
    tr.update(np.array(["a"] * 4), np.array([5.0, 5.0, 5.0, 5.0]))
    assert tr.get_stats()["a"]["count"] == 4 and tr.get_stats()["a"]["mean"] == 5.0  # ring buffer of 4
    np.testing.assert_allclose(global_advantages(r), (r - r.mean()) / r.std())


def test_parser_prompts_callbacks():
    from ddpo_b200.training import callback_fns, evaluate_callbacks, make_prompts
    from ddpo_b200.utils.parser import Parser
    a = Parser().parse_args("pg", ["--dataset", "compressed-animals", "--ppo_clip_range", "2e-4", "--seed", "3"])
    assert a.filter_field == "jpeg" and a.ppo_clip_range == 2e-4 and a.sample_batch_size == 8 and a.seed == 3
    assert a.savepath.endswith("models/pg") and a.train_cfg is True and a.n_inference_steps == 50
    inf, tr, meta = make_prompts(a.prompt_fn, 4, identical_batch=True)
    assert len(set(inf)) == 1 and len(inf) == 4
    imgs = np.random.default_rng(0).random((2, 32, 32, 3)).astype(np.float32)
    out = evaluate_callbacks({"jpeg": callback_fns["jpeg"](), "neg": callback_fns["neg_jpeg"]()}, imgs, inf[:2], meta[:2])
    assert out["jpeg"][0].shape == (2, 1) and np.all(out["jpeg"][0] < 0)
    np.testing.assert_allclose(out["jpeg"][0], -out["neg"][0])
    assert callback_fns["arange"]()(imgs, inf[:2], meta[:2])[0].tolist() == [0, 1]


def test_rewards_take_device_cast_uint8_images():
    """the driver hands the JPEG rewards uint8 images (the reference's `(image * 255).astype(np.uint8)`, callbacks.py:181, applied
    on the device): same scores as from the float images, and `evaluate_callbacks` must not turn the bytes back into floats"""
    from ddpo_b200 import training
    rng = np.random.default_rng(0)
    imgs = rng.random((3, 32, 32, 3)).astype(np.float32)
    u8 = (imgs * 255).astype(np.uint8)
    fns = {"jpeg": training.callback_fns["jpeg"](), "neg_jpeg": training.callback_fns["neg_jpeg"]()}
    assert all(getattr(f, "accepts_uint8", False) for f in fns.values())
    a = training.evaluate_callbacks(fns, imgs, ["a", "b", "c"], [{}] * 3)
    b = training.evaluate_callbacks(fns, u8, ["a", "b", "c"], [{}] * 3)
    for k in fns:
        assert np.array_equal(a[k][0], b[k][0])
    assert not getattr(training.callback_fns["aesthetic"], "accepts_uint8", False)
