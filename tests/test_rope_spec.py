"""CPU: scaled rotary frequencies (kvquant_b200.rope.RotarySpec) and the argument checks of their C entry points.

* RotarySpec's inv_freq / attention_factor equal HF's bit for bit for LLaMA-3.1-8B (llama3), linear x8 (theta 1e4),
  YaRN x4 over 32768 (theta 1e6) and the default rotation: against tests/golden/rope_inv_freq.npz (written from
  transformers' ROPE_INIT_FUNCTIONS by tests/golden/gen_rope_golden.py) and, when transformers imports, live;
* length-dependent types ("dynamic", "longrope"), unknown types and malformed dicts raise;
* the *_freq attend entry points reject what their parents reject, with the parents' codes in the parents' order,
  then a missing frequency vector (KVQ_E_NULL) and a bad attention factor (KVQ_E_SHAPE); likewise the table builders
  and the decode query rotation.  Every call is rejected before anything touches a device.
"""
import ctypes
import os

import numpy as np
import pytest
import torch

import test_attend_validate as V
from kvquant_b200 import _lib
from kvquant_b200.rope import RotarySpec, resolve

HERE = os.path.dirname(os.path.abspath(__file__))
LLAMA31 = {"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
           "original_max_position_embeddings": 8192}
CASES = {
    "llama31_8b": (500000.0, LLAMA31),
    "linear8": (10000.0, {"rope_type": "linear", "factor": 8.0}),
    "yarn4": (1000000.0, {"rope_type": "yarn", "factor": 4.0, "original_max_position_embeddings": 32768}),
    "default": (10000.0, None),
}


def hf_params(theta, scaling):
    """(inv_freq, attention_factor) from transformers itself; "default" is HF's default expression (transformers 5.5's
    ROPE_INIT_FUNCTIONS has no "default" entry)."""
    if scaling is None:
        return 1.0 / (theta ** (torch.arange(0, 128, 2, dtype=torch.int64).to(dtype=torch.float) / 128)), 1.0
    from transformers import LlamaConfig
    from transformers.modeling_rope_utils import ROPE_INIT_FUNCTIONS
    params = dict(scaling, rope_theta=theta)
    cfg = LlamaConfig(hidden_size=4096, num_attention_heads=32, max_position_embeddings=131072,
                      rope_parameters=params)
    inv_freq, attn = ROPE_INIT_FUNCTIONS[scaling["rope_type"]](cfg, "cpu")
    return inv_freq.float(), float(attn)


@pytest.mark.parametrize("name", sorted(CASES))
def test_frequencies_equal_the_golden_bit_for_bit(name):
    g = np.load(os.path.join(HERE, "golden", "rope_inv_freq.npz"))
    spec = RotarySpec(*CASES[name])
    got = spec.inv_freq.numpy()
    assert got.dtype == np.float32 and got.shape == (64,)
    assert np.array_equal(got.view(np.uint32), g[name + "_inv_freq"].view(np.uint32))
    assert spec.attention_factor == float(g[name + "_attention_factor"])


@pytest.mark.parametrize("name", sorted(CASES))
def test_frequencies_equal_installed_transformers(name):
    pytest.importorskip("transformers")
    inv_freq, attn = hf_params(*CASES[name])
    spec = RotarySpec(*CASES[name])
    assert torch.equal(spec.inv_freq.view(torch.int32), inv_freq.contiguous().view(torch.int32))
    assert spec.attention_factor == attn


def test_spec_forms_and_keys():
    a = RotarySpec(500000.0, LLAMA31)
    b = RotarySpec.from_hf({"rope_theta": 500000, "rope_scaling": dict(LLAMA31, type="llama3")})
    c = RotarySpec.from_hf({"rope_parameters": dict(LLAMA31, rope_theta=500000.0)})
    assert a == b == c and hash(a) == hash(c) and a.key == c.key and a.scaled
    assert RotarySpec(1e4, {"rope_type": "linear", "factor": 8.0}) != RotarySpec(1e4, {"rope_type": "linear", "factor": 4.0})
    d = RotarySpec(1e4, {"rope_type": "default"})
    assert not d.scaled and not RotarySpec(1e4).scaled and RotarySpec.from_hf({"rope_theta": 1e4}) == RotarySpec(1e4)
    assert resolve(None, 1e4) == 1e4 and resolve(d, 5.0) == 1e4 and resolve(a, 1e4) is a
    # 35 of LLaMA-3.1's 64 pairs (every wavelength above 8192 / 4 = 2048 tokens) are lower than theta's
    base = RotarySpec(500000.0).inv_freq
    assert int((a.inv_freq < base).sum()) == 35
    assert RotarySpec(1e6, CASES["yarn4"][1]).attention_factor > 1.0


@pytest.mark.parametrize("bad,exc", [
    ({"rope_type": "dynamic", "factor": 2.0}, NotImplementedError),
    ({"rope_type": "longrope", "short_factor": [1.0], "long_factor": [1.0]}, NotImplementedError),
    ({"type": "dynamic", "factor": 2.0}, NotImplementedError),
    ({"rope_type": "ntk-by-parts", "factor": 2.0}, ValueError),
    ({"factor": 8.0}, ValueError),                                              # no type
    ({"rope_type": "linear"}, ValueError),                                      # no factor
    ({"rope_type": "linear", "factor": 0.0}, ValueError),
    ({"rope_type": "linear", "factor": float("nan")}, ValueError),
    ({"rope_type": "linear", "factor": "8"}, ValueError),
    ({"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0}, ValueError),
    ({"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 4.0, "high_freq_factor": 1.0,
      "original_max_position_embeddings": 8192}, ValueError),
    ({"rope_type": "yarn", "factor": 4.0}, ValueError),
    ({"rope_type": "linear", "factor": 2.0, "partial_rotary_factor": 0.5}, ValueError),
])
def test_rejected_scalings_raise(bad, exc):
    with pytest.raises(exc):
        RotarySpec(1e4, bad)


def test_malformed_configs_raise():
    with pytest.raises(ValueError):
        RotarySpec(0.5)
    with pytest.raises(ValueError):
        RotarySpec.from_hf({"rope_theta": 1e4, "rope_scaling": "linear"})
    with pytest.raises(ValueError):
        RotarySpec.from_hf({"rope_parameters": ["linear"]})
    with pytest.raises(TypeError):
        resolve(10000.0, 1e4)
    with pytest.raises(NotImplementedError, match="sequence length"):
        RotarySpec.from_hf({"rope_theta": 1e4, "rope_scaling": {"rope_type": "dynamic", "factor": 2.0}})


# ---- the *_freq entry points: the parent's checks, then the new ones ---------------------------------------------------
FREQ_OF = {"kvq_attend_gqa": "kvq_attend_gqa_freq", "kvq_attend_gqa_dyn": "kvq_attend_gqa_dyn_freq",
           "kvq_attend_batch": "kvq_attend_batch_freq", "kvq_attend_paged": "kvq_attend_paged_freq"}


def call_freq(fn, freq=V.P, attn=1.0, **kw):
    """V.call with `fn`'s *_freq sibling: (rope_freq, attn_factor) in place of theta."""
    lib = _lib.load()
    parent = getattr(lib, fn)
    sib = getattr(lib, FREQ_OF[fn])

    class Shim:   # V.call looks the entry point up by name; splice (freq, attn) where theta (10000.0) goes
        def __getattr__(self, name):
            assert name == fn

            def f(*args):
                i = [k for k, a in enumerate(args) if isinstance(a, float) and a == 10000.0]
                assert len(i) == 1
                return sib(*args[:i[0]], freq, attn, *args[i[0] + 1:])
            return f
    real = _lib.load
    _lib.load = lambda: Shim()
    try:
        return V.call(fn, **kw)
    finally:
        _lib.load = real
        assert parent is not None


PARENT_CASES = [dict(pos=-1), dict(pos=-1, L=100, npos=99), dict(kcache=V.ODD), dict(scratch=V.ODD), dict(bits=5),
                dict(bits=1), dict(kcache=V.ODD, bits=5), dict(q=None), dict(out=None), dict(rope=None),
                dict(Hq=30, Hkv=30), dict(Hq=68, Hkv=68), dict(L=644), dict(n_sink=65, sink_k=V.P, sink_v=V.P),
                dict(n_sink=2), dict(ko=V.P), dict(voi=V.P), dict(ko=V.P, koi=V.P, n_out=0), dict(npos=639),
                dict(vcache=V.ODD), dict(Hq=32, Hkv=12), dict(Hq=32, Hkv=6), dict(Hq=32, Hkv=0), dict(vcent=None),
                dict(rope_half=V.P), dict(bits=5, q=None), dict(bits=5, L=644), dict(kcache=V.ODD, ko=V.P),
                dict(len_dev=None), dict(L=0), dict(B=0), dict(B=257), dict(vcent=None, q=None), dict(table=None),
                dict(page=100), dict(n_pool=0)]


@pytest.mark.parametrize("fn", sorted(FREQ_OF))
def test_freq_entry_points_keep_the_parent_codes_then_check_the_frequencies(fn):
    for kw in PARENT_CASES:   # only inputs the parent rejects: nothing here may reach a launch
        if ("table" in kw or "page" in kw or "n_pool" in kw) and fn != "kvq_attend_paged":
            continue
        if "B" in kw and fn not in V.BATCHED or "len_dev" in kw and fn == "kvq_attend_gqa":
            continue
        want = V.call(fn, **kw)
        assert want < 0, (fn, kw)
        # the parent's fault wins over a missing vector or a bad factor
        for extra in (dict(), dict(freq=None), dict(attn=0.0)):
            assert call_freq(fn, **extra, **kw) == want, (fn, kw, extra)
    assert call_freq(fn, freq=None) == V.E_NULL
    for bad in (0.0, -1.0, float("inf"), float("nan")):
        assert call_freq(fn, attn=bad) == V.E_SHAPE
    assert call_freq(fn, freq=None, attn=0.0) == V.E_NULL


def test_table_builders_and_query_rotation_checks():
    lib = _lib.load()
    P = V.P
    for fn in (lib.kvq_rope_table_build_freq, lib.kvq_rope_table_build_freq_half):
        assert fn(None, P, 1.0, 4096, None) == V.E_NULL and fn(P, None, 1.0, 4096, None) == V.E_NULL
        assert fn(P, P, 1.0, 0, None) == V.E_SHAPE and fn(P, P, 1.0, (1 << 30) + 1, None) == V.E_SHAPE
        assert fn(P, P, 0.0, 4096, None) == V.E_SHAPE and fn(P, P, float("nan"), 4096, None) == V.E_SHAPE
    f = lib.kvq_dec_rope_split_freq
    assert f(None, P, 1.0, None, 0, P, P, P, 32, 8, 1, None) == V.E_NULL
    assert f(P, None, 1.0, None, 0, P, P, P, 32, 8, 1, None) == V.E_NULL
    assert f(P, P, 1.0, None, 0, P, P, P, 32, 12, 1, None) == V.E_SHAPE
    assert f(P, P, 1.0, None, 0, P, P, P, 32, 8, 0, None) == V.E_SHAPE
    assert f(P, P, 0.0, None, 0, P, P, P, 32, 8, 1, None) == V.E_SHAPE


def test_harness_scoping():
    from kvquant_b200 import decode as kd
    cfg = kd.DecodeConfig.llama31_8b()
    assert (cfg.n_heads, cfg.kv_heads, cfg.rope_theta) == (32, 8, 500000.0)
    assert cfg.rotary == RotarySpec(500000.0, LLAMA31)
    assert kd.DecodeConfig.llama3_8b().rotary is None and kd.DecodeConfig.llama7b().rotary is None
    with pytest.raises(NotImplementedError):
        kd.DecoderStage(kd.DecodeConfig.llama31_8b(n_kv_heads=None), 0, 1, "cpu", None, sp=(0, 2))
