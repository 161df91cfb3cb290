"""Rotary position embeddings: the frequencies the quantised cache's readers rotate keys and queries with.

The cache stores pre-RoPE keys, so every reader rotates them at read time from a cos / sin table.  A plain
`rope_theta` float gives the LLaMA-2 table, f_j = theta^(-2j/128).  Models that reach long contexts by scaling RoPE
(HF `rope_scaling` / `rope_parameters` with rope_type "linear", "llama3" or "yarn") have other per-pair frequencies
and, for YaRN, an attention factor that multiplies cos and sin of queries and keys alike.  `RotarySpec` describes
either, and computes HF's `inv_freq` and `attention_factor` itself (the formulas of
transformers.modeling_rope_utils.ROPE_INIT_FUNCTIONS restated in the same fp32 operations, head_dim 128), so that the
library does not import transformers at run time.  DESIGN.md section 4.13.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

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
        raise NotImplementedError("rope_type %r is not supported: %s, and the quantised cache's readers use one "
                                  "static table per model" % (t, _LENGTH_DEPENDENT[t]))
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
        return cls(theta, scaling)

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
    """What a reader rotates with: `rope` (a RotarySpec) when given, else the float `rope_theta`.  A spec without
    scaling becomes its float theta, so the plain-theta path (table, kernels, bits) serves it."""
    if rope is None:
        return rope_theta
    if not isinstance(rope, RotarySpec):
        raise TypeError("rope must be a RotarySpec or None, got %r" % (type(rope).__name__,))
    return rope if rope.scaled else rope.theta
