"""Writes tests/golden/rope_inv_freq.npz: HF's inv_freq (fp32 [64]) and attention_factor for the rotary specs
tests/test_rope_spec.py checks, from the installed transformers' ROPE_INIT_FUNCTIONS (CPU, offline).

    python tests/golden/gen_rope_golden.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from test_rope_spec import CASES, hf_params  # noqa: E402


def main():
    import transformers
    out = {"transformers_version": np.array(transformers.__version__)}
    for name, (theta, scaling) in CASES.items():
        inv_freq, attn = hf_params(theta, scaling)
        out[name + "_inv_freq"] = inv_freq.numpy().astype(np.float32)
        out[name + "_attention_factor"] = np.float64(attn)
    np.savez(os.path.join(HERE, "rope_inv_freq.npz"), **out)
    print("wrote", sorted(out))


if __name__ == "__main__":
    torch.set_num_threads(1)
    main()
