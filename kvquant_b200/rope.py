"""Rotary position embeddings: the frequencies the quantised cache's readers rotate keys and queries with.

The cache stores pre-RoPE keys, so every reader rotates them at read time from a cos / sin table.  A plain
`rope_theta` float gives the LLaMA-2 table, f_j = theta^(-2j/128).  Models that reach long contexts by scaling RoPE
(HF `rope_scaling` / `rope_parameters` with rope_type "linear", "llama3" or "yarn") have other per-pair frequencies
and, for YaRN, an attention factor that multiplies cos and sin of queries and keys alike.  `RotarySpec` describes
either, and computes HF's `inv_freq` and `attention_factor` itself (the formulas of
transformers.modeling_rope_utils.ROPE_INIT_FUNCTIONS restated in the same fp32 operations, head_dim 128), so that the
library does not import transformers at run time.  DESIGN.md section 4.13.

HF's "dynamic" (dynamic NTK) and "longrope" types change their frequencies with the sequence length.
`LengthDependentRotary` describes them: its frequencies are a pure function f(s) of s, one plus the absolute position
of the last query of a call, and every reader rotates every key and the query with f(s) (DESIGN.md section 4.14).
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import torch

HEAD_DIM = 128

# Frequencies that depend on the current sequence length: the table would change as the cache grows, which one
# captured graph over a device-resident length cannot follow.
_LENGTH_DEPENDENT = {
    "dynamic": "dynamic NTK scaling changes its frequencies with the current sequence length",
    "longrope": "LongRoPE picks its frequency factors by the current sequence length",
}
_REQUIRED = {
    "default": (),
    "linear": ("factor",),
    "llama3": ("factor", "low_freq_factor", "high_freq_factor", "original_max_position_embeddings"),
    "yarn": ("factor", "original_max_position_embeddings"),
}


def _rope_type(scaling):
    t = scaling.get("rope_type", scaling.get("type"))
    if t is None:
        raise ValueError("rope scaling %r names no rope_type" % (scaling,))
    if t in _LENGTH_DEPENDENT:
        raise NotImplementedError("rope_type %r is not supported by RotarySpec: %s, and RotarySpec's readers use one "
                                  "static table per model (use LengthDependentRotary)" % (t, _LENGTH_DEPENDENT[t]))
    if t not in _REQUIRED:
        raise ValueError("unknown rope_type %r (supported: %s)" % (t, ", ".join(sorted(_REQUIRED))))
    return t


def _default_inv_freq(base):
    return 1.0 / (base ** (torch.arange(0, HEAD_DIM, 2, dtype=torch.int64).to(dtype=torch.float) / HEAD_DIM))


@dataclass(frozen=True)
class RotarySpec:
    """theta (the rope base) and optionally HF's rope scaling dict.  Hashable; `key` names its table.

    A spec without scaling, or with rope_type "default", is the plain-theta rotation: the readers take the theta path
    (its table, its kernels, its bits), exactly as if `rope_theta=theta` had been passed."""
    theta: float
    scaling: tuple = None        # sorted (key, value) items of the scaling dict; pass a dict, it is frozen here

    def __post_init__(self):
        theta = float(self.theta)
        if not (theta > 1.0 and math.isfinite(theta)):
            raise ValueError("rope theta must be a finite number > 1, got %r" % (self.theta,))
        object.__setattr__(self, "theta", theta)
        sc = self.scaling
        if sc is None:
            return
        sc = dict(sc)
        t = _rope_type(sc)
        for k in _REQUIRED[t]:
            v = sc.get(k)
            if isinstance(v, bool) or not isinstance(v, (int, float)) or not (v > 0 and math.isfinite(v)):
                raise ValueError("rope_type %r needs a positive number %r, got %r" % (t, k, v))
        if t == "llama3" and not sc["high_freq_factor"] > sc["low_freq_factor"]:
            raise ValueError("llama3 scaling needs high_freq_factor > low_freq_factor")
        prf = sc.get("partial_rotary_factor", 1.0)
        if prf != 1.0:
            raise ValueError("partial_rotary_factor %r: every rotary pair of the 128-wide head is rotated here" % prf)
        sc.pop("type", None)
        sc["rope_type"] = t
        sc.pop("rope_theta", None)
        object.__setattr__(self, "scaling", tuple(sorted(sc.items())))

    @classmethod
    def from_hf(cls, config):
        """From an HF model config dict (or object): rope_theta plus rope_scaling (transformers 4.x) or
        rope_parameters (5.x, which also carries rope_theta)."""
        return cls(*_hf_theta_scaling(config)[:2])

    @property
    def rope_type(self):
        return "default" if self.scaling is None else dict(self.scaling)["rope_type"]

    @property
    def scaled(self):
        """False for the plain-theta rotation (no scaling, or rope_type "default")."""
        return self.rope_type != "default"

    @property
    def key(self):
        return (self.theta, self.scaling)

    @property
    def inv_freq(self):
        """HF's inv_freq: f32 [64] on the CPU."""
        return self._params()[0].clone()

    @property
    def attention_factor(self):
        """HF's attention_factor (1.0 except for YaRN): multiplies cos and sin of queries and keys."""
        return self._params()[1]

    def _params(self):
        cached = self.__dict__.get("_cache")
        if cached is None:
            cached = _compute(self.theta, self.rope_type, dict(self.scaling or ()))
            object.__setattr__(self, "_cache", cached)
        return cached


def _hf_theta_scaling(config):
    """(rope_theta, scaling dict or None, max_position_embeddings or None) of an HF config dict or object."""
    get = config.get if isinstance(config, dict) else (lambda k, d=None: getattr(config, k, d))
    params = get("rope_parameters")
    scaling = get("rope_scaling")
    if params is not None:
        if not isinstance(params, dict):
            raise ValueError("rope_parameters must be a dict, got %r" % (params,))
        theta = params.get("rope_theta", get("rope_theta"))
        scaling = params
    else:
        theta = get("rope_theta", 10000.0)
    if scaling is not None and not isinstance(scaling, dict):
        raise ValueError("rope_scaling must be a dict or None, got %r" % (scaling,))
    if theta is None:
        raise ValueError("the config names no rope_theta")
    return theta, scaling, get("max_position_embeddings")


def _positive(v):
    return not isinstance(v, bool) and isinstance(v, (int, float)) and v > 0 and math.isfinite(v)


@dataclass(frozen=True)
class LengthDependentRotary:
    """HF rope_type "dynamic" (dynamic NTK) or "longrope": frequencies that are a function f(s) of s, one plus the
    absolute position of the last query of a call.  Hashable; `key` names it.

    dynamic, M = max_position_embeddings (HF reads it from the config, not from the scaling dict): f(s) for s <= M is
    the default theta vector, bit for bit HF's; for s > M it is HF's formula base * ((factor * s / M) - (factor - 1)) **
    (128 / 126), then 1 / base' ** (2j / 128), evaluated in float64 and rounded once to fp32 (the device computes the
    same in double precision).  attention_factor 1.
    longrope: 1 / (short_factor * theta ** (2j / 128)) for s <= original_max_position_embeddings, long_factor above,
    both in HF's fp32 operations (bit for bit); attention_factor is HF's, a constant.

    f is a pure function of s.  HF's module keeps state instead (it grows max_seq_len_cached and resets only below M);
    that history is not reproduced: a decode attend at s equals the attention of HF's uncached forward over the first
    s positions at its last query."""
    theta: float
    scaling: tuple                 # sorted (key, value) items of the scaling dict; pass a dict, it is frozen here
    max_position_embeddings: int

    def __post_init__(self):
        theta = float(self.theta)
        if not (theta > 1.0 and math.isfinite(theta)):
            raise ValueError("rope theta must be a finite number > 1, got %r" % (self.theta,))
        object.__setattr__(self, "theta", theta)
        M = self.max_position_embeddings
        if isinstance(M, bool) or not isinstance(M, int) or M <= 0:
            raise ValueError("max_position_embeddings must be a positive int, got %r" % (M,))
        if not isinstance(self.scaling, (dict, tuple, list)):
            raise ValueError("scaling must be a dict, got %r" % (self.scaling,))
        sc = dict(self.scaling)
        t = sc.get("rope_type", sc.get("type"))
        if t not in _LENGTH_DEPENDENT:
            raise ValueError("LengthDependentRotary takes rope_type 'dynamic' or 'longrope', got %r" % (t,))
        prf = sc.get("partial_rotary_factor", 1.0)
        if prf != 1.0:
            raise ValueError("partial_rotary_factor %r: every rotary pair of the 128-wide head is rotated here" % prf)
        if t == "dynamic":
            if not _positive(sc.get("factor")):
                raise ValueError("rope_type 'dynamic' needs a positive number 'factor', got %r" % (sc.get("factor"),))
        else:
            om = sc.get("original_max_position_embeddings")
            if isinstance(om, bool) or not isinstance(om, int) or om <= 0:
                raise ValueError("rope_type 'longrope' needs a positive int 'original_max_position_embeddings', got %r"
                                 % (om,))
            for k in ("short_factor", "long_factor"):
                v = sc.get(k)
                if (not isinstance(v, (list, tuple)) or len(v) != HEAD_DIM // 2
                        or not all(_positive(x) for x in v)):
                    raise ValueError("rope_type 'longrope' needs %r: a list of %d finite positive numbers"
                                     % (k, HEAD_DIM // 2))
                sc[k] = tuple(float(x) for x in v)
            for k in ("factor", "attention_factor"):
                if sc.get(k) is not None and not _positive(sc[k]):
                    raise ValueError("rope_type 'longrope': %r must be a positive number, got %r" % (k, sc[k]))
        sc.pop("type", None)
        sc["rope_type"] = t
        sc.pop("rope_theta", None)
        object.__setattr__(self, "scaling", tuple(sorted(sc.items())))

    @classmethod
    def from_hf(cls, config):
        """From an HF model config dict (or object): rope_theta, max_position_embeddings and rope_scaling
        (transformers 4.x) or rope_parameters (5.x)."""
        theta, scaling, M = _hf_theta_scaling(config)
        if scaling is None:
            raise ValueError("the config names no rope scaling")
        if M is None:
            raise ValueError("the config names no max_position_embeddings")
        return cls(theta, scaling, M)

    @property
    def rope_type(self):
        return self._p["rope_type"]

    @property
    def key(self):
        return ("length", self.theta, self.scaling, self.max_position_embeddings)

    @property
    def _p(self):
        return dict(self.scaling)

    @property
    def switch_position(self):
        """The largest s served by the first frequency vector: M (dynamic) or original_max_position_embeddings."""
        p = self._p
        return self.max_position_embeddings if p["rope_type"] == "dynamic" else p["original_max_position_embeddings"]

    @property
    def attention_factor(self):
        p = self._p
        if p["rope_type"] == "dynamic":
            return 1.0
        if p.get("attention_factor") is not None:
            return float(p["attention_factor"])
        factor = p.get("factor")
        if factor is None:
            factor = self.max_position_embeddings / p["original_max_position_embeddings"]
        if factor <= 1.0:
            return 1.0
        return math.sqrt(1 + math.log(factor) / math.log(p["original_max_position_embeddings"]))

    def base_vectors(self):
        """(f_lo, f_hi) f32 [64] on the CPU: the default vector and None (dynamic), or the short and long vectors."""
        cached = self.__dict__.get("_vec")
        if cached is None:
            p = self._p
            if p["rope_type"] == "dynamic":
                cached = (_default_inv_freq(self.theta), None)
            else:
                shape = torch.arange(0, HEAD_DIM, 2, dtype=torch.int64).float() / HEAD_DIM
                cached = tuple(1.0 / (torch.tensor(p[k], dtype=torch.float32) * self.theta ** shape)
                               for k in ("short_factor", "long_factor"))
            object.__setattr__(self, "_vec", cached)
        return cached

    def inv_freq_at(self, s):
        """f(s): f32 [64] on the CPU (s = one plus the absolute position of the last query)."""
        s = int(s)
        lo, hi = self.base_vectors()
        if s <= self.switch_position:
            return lo.clone()
        if hi is not None:
            return hi.clone()
        p, M = self._p, self.max_position_embeddings
        factor = float(p["factor"])
        base = self.theta * ((factor * s / M) - (factor - 1)) ** (HEAD_DIM / (HEAD_DIM - 2))
        e = np.arange(0, HEAD_DIM, 2, dtype=np.float64) / HEAD_DIM
        return torch.from_numpy((1.0 / np.float64(base) ** e).astype(np.float32))

    def device_params(self):
        """(mode, (theta, factor), switch position) of kvq_rope_len_update."""
        p = self._p
        if p["rope_type"] == "dynamic":
            return 0, (self.theta, float(p["factor"])), self.max_position_embeddings
        return 1, (self.theta, 1.0), p["original_max_position_embeddings"]


def _compute(base, t, p):
    """(inv_freq f32 [64], attention_factor): modeling_rope_utils' formulas for head_dim 128, same fp32 operations."""
    dim = HEAD_DIM
    if t == "default":
        return _default_inv_freq(base), 1.0
    if t == "linear":
        inv_freq = _default_inv_freq(base)
        inv_freq /= p["factor"]
        return inv_freq, 1.0
    if t == "llama3":
        inv_freq = _default_inv_freq(base)
        factor, low, high = p["factor"], p["low_freq_factor"], p["high_freq_factor"]
        old_context_len = p["original_max_position_embeddings"]
        low_freq_wavelen = old_context_len / low
        high_freq_wavelen = old_context_len / high
        wavelen = 2 * math.pi / inv_freq
        inv_freq_llama = torch.where(wavelen > low_freq_wavelen, inv_freq / factor, inv_freq)
        smooth_factor = (old_context_len / wavelen - low) / (high - low)
        smoothed_inv_freq = (1 - smooth_factor) * inv_freq_llama / factor + smooth_factor * inv_freq_llama
        is_medium_freq = ~(wavelen < high_freq_wavelen) * ~(wavelen > low_freq_wavelen)
        return torch.where(is_medium_freq, smoothed_inv_freq, inv_freq_llama), 1.0
    assert t == "yarn"
    factor = p["factor"]
    attention_factor = p.get("attention_factor")
    mscale, mscale_all_dim = p.get("mscale"), p.get("mscale_all_dim")
    original_max = p["original_max_position_embeddings"]

    def get_mscale(scale, m=1):
        return 1.0 if scale <= 1 else 0.1 * m * math.log(scale) + 1.0

    if attention_factor is None:
        if mscale and mscale_all_dim:
            attention_factor = float(get_mscale(factor, mscale) / get_mscale(factor, mscale_all_dim))
        else:
            attention_factor = get_mscale(factor)
    beta_fast = p.get("beta_fast") or 32
    beta_slow = p.get("beta_slow") or 1

    def correction_dim(num_rotations):
        return (dim * math.log(original_max / (num_rotations * 2 * math.pi))) / (2 * math.log(base))

    lo, hi = correction_dim(beta_fast), correction_dim(beta_slow)
    if p.get("truncate", True):
        lo, hi = math.floor(lo), math.ceil(hi)
    lo, hi = max(lo, 0), min(hi, dim - 1)
    if lo == hi:
        hi += 0.001
    ramp = torch.clamp((torch.arange(dim // 2, dtype=torch.float32) - lo) / (hi - lo), 0, 1)
    pos_freqs = base ** (torch.arange(0, dim, 2).to(dtype=torch.float) / dim)
    inv_freq_extrapolation = 1.0 / pos_freqs
    inv_freq_interpolation = 1.0 / (factor * pos_freqs)
    extrapolation_factor = 1 - ramp
    inv_freq = inv_freq_interpolation * (1 - extrapolation_factor) + inv_freq_extrapolation * extrapolation_factor
    return inv_freq, float(attention_factor)


def resolve(rope, rope_theta):
    """What a reader rotates with: `rope` (a RotarySpec or LengthDependentRotary) when given, else the float
    `rope_theta`.  A spec without scaling becomes its float theta, so the plain-theta path (table, kernels, bits)
    serves it."""
    if rope is None:
        return rope_theta
    if isinstance(rope, LengthDependentRotary):
        return rope
    if not isinstance(rope, RotarySpec):
        raise TypeError("rope must be a RotarySpec, a LengthDependentRotary or None, got %r" % (type(rope).__name__,))
    return rope if rope.scaled else rope.theta
