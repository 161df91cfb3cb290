"""CPU: length-dependent rotary frequencies (kvquant_b200.rope.LengthDependentRotary, DESIGN.md section 4.14).

* f(s) = inv_freq_at(s) against HF's for two dynamic NTK specs and one LongRoPE spec, at every s in [M - 4, M + 4096],
  the powers of two up to 2^20 and seeded samples: against tests/golden/rope_len_inv_freq.npz (written from
  transformers by tests/golden/gen_rope_len_golden.py) and, when transformers imports, live.  Dynamic s <= M and both
  LongRoPE vectors are bit for bit; dynamic s > M (float64 evaluation of HF's formula, rounded once to fp32) is within
  ULP_BOUND of HF's fp32 tensor branch (the one HF's dynamic_rope_update calls), the largest difference found here;
  The fixture holds HF's bits losslessly but small: the vector(s) below the switch, which LongRoPE vector each length
  got, and for dynamic s > M the signed ulp difference of HF's bits from golden_baseline(s) (decode_golden rebuilds
  the rows);
* from_hf, validation errors, resolve() and the decode config;
* kvq_rope_len_update, kvq_attend_{batch,paged}_freq_seq and kvq_dec_rope_split_freq_seq reject bad arguments before
  anything touches a device.
"""
import ctypes
import os

import numpy as np
import pytest
import torch

import test_attend_validate as V
from kvquant_b200 import _lib
from kvquant_b200.rope import LengthDependentRotary, RotarySpec, resolve

HERE = os.path.dirname(os.path.abspath(__file__))
ULP_BOUND = 3
LONG = [1.0 + 0.03125 * i for i in range(64)]
SHORT = [1.0 + 0.0078125 * (i % 7) for i in range(64)]
CASES = {
    "dyn_1e4": (10000.0, {"rope_type": "dynamic", "factor": 2.0}, 4096),
    "dyn_1e6": (1000000.0, {"rope_type": "dynamic", "factor": 4.0}, 32768),
    "longrope": (10000.0, {"rope_type": "longrope", "long_factor": LONG, "short_factor": SHORT,
                           "original_max_position_embeddings": 4096}, 131072),
}


def lengths(M):
    rng = np.random.default_rng(M)
    s = set(range(M - 4, M + 4097)) | {2 ** k for k in range(21)} | set(rng.integers(1, 1 << 20, 64).tolist())
    return np.array(sorted(s), dtype=np.int64)


def hf_inv_freq(theta, scaling, M, s):
    """HF's (inv_freq, attention_factor) at sequence length s; dynamic through the tensor branch of
    dynamic_rope_update."""
    from transformers import LlamaConfig
    from transformers.modeling_rope_utils import ROPE_INIT_FUNCTIONS
    cfg = LlamaConfig(hidden_size=4096, num_attention_heads=32, max_position_embeddings=M,
                      rope_parameters=dict(scaling, rope_theta=theta))
    t = scaling["rope_type"]
    arg = torch.tensor(int(s)) if t == "dynamic" else int(s)
    f, a = ROPE_INIT_FUNCTIONS[t](cfg, "cpu", seq_len=arg)
    return f.float(), float(a)


def golden_baseline(theta, factor, M, s):
    """HF's dynamic formula for s > M in float64 (Python floats, C pow), rounded once to fp32: the rows the fixture
    stores HF's bits against."""
    base = theta * ((factor * s / M) - (factor - 1)) ** (128 / 126)
    return np.array([1.0 / base ** (2 * j / 128) for j in range(64)], dtype=np.float64).astype(np.float32)


def encode_golden(name, ss, rows):
    """The fixture entries of one case from HF's rows [N, 64] at lengths ss (what decode_golden inverts)."""
    theta, scaling, M = CASES[name]
    rows = np.asarray(rows, dtype=np.float32)
    out = {name + "_s": ss}
    if scaling["rope_type"] == "longrope":
        sw = scaling["original_max_position_embeddings"]
        lo, hi = rows[ss <= sw][0], rows[ss > sw][0]
        which = np.array([0 if np.array_equal(r.view(np.int32), lo.view(np.int32)) else 1 for r in rows], np.uint8)
        vecs = np.stack([lo, hi])
        assert np.array_equal(vecs[which].view(np.int32), rows.view(np.int32))
        out.update({name + "_vectors": vecs, name + "_which": which})
        return out
    below = ss <= M
    lo = rows[below][0]
    assert all(np.array_equal(r.view(np.int32), lo.view(np.int32)) for r in rows[below])
    base = np.stack([golden_baseline(theta, scaling["factor"], M, int(x)) for x in ss[~below]])
    d = rows[~below].view(np.int32).astype(np.int64) - base.view(np.int32).astype(np.int64)
    assert np.abs(d).max() < 127
    out.update({name + "_default": lo, name + "_ulp_above": d.astype(np.int8)})
    return out


def decode_golden(g, name):
    """(lengths, HF's rows [N, 64] f32) of one case of the fixture, bit for bit."""
    theta, scaling, M = CASES[name]
    ss = g[name + "_s"]
    if scaling["rope_type"] == "longrope":
        return ss, g[name + "_vectors"][g[name + "_which"]]
    rows = np.empty((len(ss), 64), dtype=np.float32)
    below = ss <= M
    rows[below] = g[name + "_default"]
    base = np.stack([golden_baseline(theta, scaling["factor"], M, int(x)) for x in ss[~below]])
    rows[~below] = (base.view(np.int32).astype(np.int64) + g[name + "_ulp_above"]).astype(np.int32).view(np.float32)
    return ss, rows


def _ulps(a, b):
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


def _check(name, ss, ref):
    theta, scaling, M = CASES[name]
    spec = LengthDependentRotary(theta, scaling, M)
    sw = spec.switch_position
    worst = 0
    for s, r in zip(ss, ref):
        mine = spec.inv_freq_at(int(s)).numpy()
        if scaling["rope_type"] == "longrope" or s <= sw:
            assert np.array_equal(mine.view(np.int32), r.view(np.int32)), (name, int(s))
        else:
            worst = max(worst, int(_ulps(mine, r).max()))
    assert worst <= ULP_BOUND, (name, worst)
    return worst


@pytest.mark.parametrize("name", sorted(CASES))
def test_inv_freq_at_matches_the_golden_fixture(name):
    g = np.load(os.path.join(HERE, "golden", "rope_len_inv_freq.npz"))
    ss, rows = decode_golden(g, name)
    assert np.array_equal(ss, lengths(CASES[name][2] if name != "longrope" else 4096))
    _check(name, ss, rows)
    spec = LengthDependentRotary(*CASES[name])
    assert spec.attention_factor == float(g[name + "_attention_factor"])


@pytest.mark.parametrize("name", sorted(CASES))
def test_inv_freq_at_matches_transformers_live(name):
    pytest.importorskip("transformers")
    theta, scaling, M = CASES[name]
    ss = lengths(M if name != "longrope" else 4096)[::37]
    ref = []
    for s in ss:
        f, a = hf_inv_freq(theta, scaling, M, s)
        ref.append(f.numpy())
        assert a == LengthDependentRotary(theta, scaling, M).attention_factor
    _check(name, ss, ref)


def test_dynamic_below_the_switch_is_the_default_vector_and_host_f_is_pure():
    theta, scaling, M = CASES["dyn_1e6"]
    spec = LengthDependentRotary(theta, scaling, M)
    default = RotarySpec(theta).inv_freq
    for s in (1, 2, M - 1, M):
        assert torch.equal(spec.inv_freq_at(s), default)
    a = spec.inv_freq_at(M + 10)
    spec.inv_freq_at(3 * M)
    assert torch.equal(spec.inv_freq_at(M + 10), a)        # no history
    assert not torch.equal(a, default)


def test_from_hf_reads_both_config_forms_and_max_position_embeddings():
    old = {"rope_theta": 1e6, "max_position_embeddings": 32768, "rope_scaling": {"type": "dynamic", "factor": 4.0}}
    new = {"max_position_embeddings": 32768, "rope_parameters": {"rope_type": "dynamic", "factor": 4.0,
                                                                  "rope_theta": 1e6}}
    a, b = LengthDependentRotary.from_hf(old), LengthDependentRotary.from_hf(new)
    assert a == b and hash(a) == hash(b) and a.key == b.key and a.rope_type == "dynamic"
    assert a == LengthDependentRotary(*CASES["dyn_1e6"])
    lr = LengthDependentRotary.from_hf({"rope_theta": 1e4, "max_position_embeddings": 131072,
                                        "rope_scaling": CASES["longrope"][1]})
    assert lr.rope_type == "longrope" and lr.attention_factor > 1.0
    with pytest.raises(ValueError, match="max_position_embeddings"):
        LengthDependentRotary.from_hf({"rope_theta": 1e4, "rope_scaling": {"type": "dynamic", "factor": 2.0}})


@pytest.mark.parametrize("bad, match", [
    (dict(scaling={"rope_type": "dynamic"}), "factor"),
    (dict(scaling={"rope_type": "dynamic", "factor": 0.0}), "factor"),
    (dict(scaling={"rope_type": "dynamic", "factor": 2.0}, M=0), "max_position_embeddings"),
    (dict(scaling={"rope_type": "dynamic", "factor": 2.0}, M=-5), "max_position_embeddings"),
    (dict(scaling={"rope_type": "dynamic", "factor": 2.0, "partial_rotary_factor": 0.5}), "partial_rotary_factor"),
    (dict(scaling=dict(CASES["longrope"][1], long_factor=LONG[:63])), "long_factor"),
    (dict(scaling=dict(CASES["longrope"][1], short_factor=SHORT[:-1] + [float("inf")])), "short_factor"),
    (dict(scaling=dict(CASES["longrope"][1], short_factor=SHORT[:-1] + [-1.0])), "short_factor"),
    (dict(scaling={k: v for k, v in CASES["longrope"][1].items() if k != "original_max_position_embeddings"}),
     "original_max_position_embeddings"),
    (dict(scaling={"rope_type": "llama3", "factor": 8.0}), "dynamic"),
])
def test_validation_errors(bad, match):
    with pytest.raises(ValueError, match=match):
        LengthDependentRotary(1e4, bad["scaling"], bad.get("M", 4096))


def test_rotary_spec_still_refuses_and_resolve_accepts_the_new_type():
    with pytest.raises(NotImplementedError, match="sequence length"):
        RotarySpec(1e4, {"rope_type": "dynamic", "factor": 2.0})
    spec = LengthDependentRotary(*CASES["dyn_1e4"])
    assert resolve(spec, 10000.0) is spec


def test_decode_config_builds_the_new_type():
    from kvquant_b200.decode import DecodeConfig
    cfg = DecodeConfig.llama3_8b(rope_scaling={"rope_type": "dynamic", "factor": 4.0}, max_position_embeddings=8192)
    assert cfg.rotary == LengthDependentRotary(500000.0, {"rope_type": "dynamic", "factor": 4.0}, 8192)
    with pytest.raises(ValueError, match="max_position_embeddings"):
        DecodeConfig.llama3_8b(rope_scaling={"rope_type": "dynamic", "factor": 4.0}).rotary
    assert DecodeConfig.llama31_8b().rotary.rope_type == "llama3"


# -- argument codes of the new entry points: rejected before any launch -----------------------------------------
NULL, SHAPE = -3, -2
P = 4096


def _update(lib, **kw):
    params = np.array([1e4, 2.0], dtype=np.float64)
    a = dict(mode=0, params=params.ctypes.data, m_pos=4096, f_lo=P, f_hi=None, attn=1.0, s=10, len_dev=None,
             len_add=0, L_cap=0, pos_offset=0, B=1, f_cur=P, state=P, table=P, npos=8192)
    a.update(kw)
    return lib.kvq_rope_len_update(a["mode"], a["params"], a["m_pos"], a["f_lo"], a["f_hi"], a["attn"], a["s"],
                                   a["len_dev"], a["len_add"], a["L_cap"], a["pos_offset"], a["B"], a["f_cur"],
                                   a["state"], a["table"], a["npos"], None)


def test_rope_len_update_argument_codes():
    lib = _lib.load()
    for k in ("params", "f_lo", "f_cur", "state", "table"):
        assert _update(lib, **{k: None}) == NULL, k
    assert _update(lib, mode=1) == NULL                         # LongRoPE needs f_hi
    bad_theta = np.array([1.0, 2.0], dtype=np.float64)
    bad_factor = np.array([1e4, 0.0], dtype=np.float64)
    for kw in (dict(mode=2), dict(m_pos=0), dict(npos=0), dict(npos=(1 << 30) + 1), dict(B=0), dict(B=257),
               dict(attn=0.0), dict(attn=float("inf")), dict(params=bad_theta.ctypes.data),
               dict(params=bad_factor.ctypes.data), dict(s=-1), dict(s=8193), dict(B=2),
               dict(len_dev=P, L_cap=-1), dict(len_dev=P, pos_offset=-1), dict(len_dev=P, L_cap=8192, pos_offset=1)):
        assert _update(lib, **kw) == SHAPE, kw
    assert _update(lib, mode=1, f_hi=P, params=bad_factor.ctypes.data, s=-1) == SHAPE   # factor unused by LongRoPE


def test_dec_rope_split_freq_seq_argument_codes():
    lib = _lib.load()
    f = lib.kvq_dec_rope_split_freq_seq
    assert f(None, P, 1.0, None, 0, P, P, P, 32, 8, 1, None) == NULL
    assert f(P, None, 1.0, None, 0, P, P, P, 32, 8, 1, None) == NULL
    assert f(P, P, 1.0, None, 0, P, P, P, 32, 8, 0, None) == SHAPE
    assert f(P, P, 0.0, None, 0, P, P, P, 32, 8, 1, None) == SHAPE
    assert f(P, P, 1.0, None, 0, P, P, P, 30, 8, 1, None) == SHAPE


@pytest.mark.parametrize("fn", ["kvq_attend_batch_freq_seq", "kvq_attend_paged_freq_seq"])
def test_per_sequence_attend_entry_points_share_their_parents_codes(fn):
    """Each call differs from its *_freq parent only in the name: the parent's code comes back."""
    lib = _lib.load()
    parent = getattr(lib, fn.replace("_seq", ""))
    child = getattr(lib, fn)
    nargs = len(_lib.SIGNATURES[fn][1])
    types = _lib.SIGNATURES[fn][1]
    base = [P if t is ctypes.c_void_p else (1.0 if t is ctypes.c_float else 1) for t in types]
    # bits=9 -> KVQ_E_BITS after the batch shape checks; B=0 -> KVQ_E_SHAPE; q=None ... -> KVQ_E_NULL
    for patch in ({0: 9}, {1: 0}, {2: None}, {1: 300}):
        args = list(base)
        for i, v in patch.items():
            args[i] = v
        assert child(*args) == parent(*args) != 0, (fn, patch)
    assert nargs == len(_lib.SIGNATURES[fn.replace("_seq", "")][1])
