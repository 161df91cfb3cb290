"""Generates tests/golden/quantizers_b{4,3}.pkl by running the REFERENCE's own calibration code
(quant/kvquant/simquant_module_quantizer.py: SimQuant.add_batch + SimQuant.quantize, the functions
quant/llama_simquant.py:275 calls to fill quantizers.pickle) on small synthetic activations, on the CPU.

    python tests/golden/gen_quantizers_golden.py        # needs a reference checkout (oracle/build_ref.py: REF_ROOT)

The fixtures hold plain numpy arrays / floats in the reference's tuple layout, so the tests need neither torch
pickles nor the reference at run time.

Q-Norm: the reference's own `quantize(norm=True)` cannot run -- it calls `round_to_nearest_pole_sim(...,
return_freq=True)` (simquant_module_quantizer.py:542), a keyword that function does not have (line 10).  The `_norm`
fixtures therefore carry the reference-produced (upper, lower, centroids) plus a (normscale, normoffset) pair computed
here with the formulas of lines 536-548 (mean / std matching of the rounded values)."""
import os
import pickle
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))), "oracle"))
from build_ref import REF_ROOT  # noqa: E402
sys.path.insert(0, os.path.join(REF_ROOT, "quant"))
from kvquant.simquant_module_quantizer import SimQuant  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
HIDDEN, TOKENS, LAYERS = 512, 768, 2


def acts(seed, per_token):
    g = np.random.default_rng(seed)
    mu = g.normal(0, 0.5, HIDDEN)
    sd = np.exp(g.normal(0, 0.5, HIDDEN))
    x = g.normal(0, 1, (TOKENS, HIDDEN)) * sd + mu
    if per_token:
        x = g.normal(0, 1, (TOKENS, HIDDEN)) * np.exp(g.normal(0, 0.3, (TOKENS, 1)))
    tail = g.random((TOKENS, HIDDEN)) < 0.005
    x[tail] += g.standard_t(3, tail.sum()) * 4
    return torch.tensor(x, dtype=torch.float32)


def qnorm_params(x, ret):
    """(normscale, normoffset) as simquant_module_quantizer.py:536-548 defines them."""
    up, lo, cent = ret[0].float(), ret[1].float(), torch.tensor(np.sort(np.asarray(ret[2][0]).ravel()), dtype=torch.float32)
    rng, zp = (up - lo) / 2, (up + lo) / 2
    a = (x - zp) / rng
    keep = ~((a > 1) | (a < -1))
    m1 = (a * keep).sum() / keep.sum()
    s1 = torch.sqrt((((a - m1) * keep) ** 2).sum() / keep.sum())
    r = cent[(a.unsqueeze(-1) - cent).abs().argmin(-1)]
    m2 = (r * keep).sum() / keep.sum()
    s2 = torch.sqrt((((r - m2) * keep) ** 2).sum() / keep.sum())
    return (s1 / s2, (-m2) * (s1 / s2) + m1)


def to_plain(ret):
    up, lo, cent = ret[0], ret[1], ret[2]
    out = [np.asarray(up, dtype=np.float32), np.asarray(lo, dtype=np.float32), [np.asarray(c, dtype=np.float32) for c in cent]]
    if len(ret) > 3:
        out += [float(ret[3]), float(ret[4])]
    return tuple(out)


def main():
    for bits in (4, 3):
        for norm in (False, True):
            q = {}
            for ln in range(LAYERS):
                for name, per_token in (("k_proj", False), ("v_proj", True)):
                    lin = torch.nn.Linear(HIDDEN, HIDDEN, bias=False)
                    sq = SimQuant(lin, bits, perchannel=True, qchannel=0)
                    sq.add_batch(None, acts(100 * ln + (7 if per_token else 3) + bits, per_token))
                    x = acts(100 * ln + (7 if per_token else 3) + bits, per_token)
                    ret = sq.quantize(include_sparse=True, sparsity_threshold=0.99, nuq=True, fisher=None, norm=False)
                    if norm:
                        ret = tuple(ret) + qnorm_params(x, ret)
                    q["model.layers.%d.self_attn.%s" % (ln, name)] = to_plain(ret)
            q["model.layers.0.self_attn.k_proj.lut"] = "skipped by deployment/llama.py:187"
            path = os.path.join(HERE, "quantizers_b%d%s.pkl" % (bits, "_norm" if norm else ""))
            with open(path, "wb") as f:
                pickle.dump(q, f, protocol=4)
            print("wrote", path, os.path.getsize(path))


if __name__ == "__main__":
    main()
