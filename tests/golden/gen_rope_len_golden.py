"""Writes tests/golden/rope_len_inv_freq.npz: HF's inv_freq (fp32 [64]) and attention_factor at every length
tests/test_rope_length_spec.py checks, for its CASES, from the installed transformers (CPU, offline).  Dynamic NTK
goes through the fp32 tensor branch that HF's dynamic_rope_update calls.  The rows are stored losslessly in the
compact form of test_rope_length_spec.encode_golden, and read back bit for bit here before the file is written.

    python tests/golden/gen_rope_len_golden.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from test_rope_length_spec import CASES, decode_golden, encode_golden, hf_inv_freq, lengths  # noqa: E402


def main():
    import transformers
    out = {"transformers_version": np.array(transformers.__version__)}
    for name, (theta, scaling, M) in CASES.items():
        ss = lengths(M if scaling["rope_type"] == "dynamic" else scaling["original_max_position_embeddings"])
        rows = [hf_inv_freq(theta, scaling, M, s) for s in ss]
        f = np.stack([r.numpy() for r, _ in rows]).astype(np.float32)
        enc = encode_golden(name, ss, f)
        back_s, back = decode_golden(enc, name)
        assert np.array_equal(back_s, ss) and np.array_equal(back.view(np.int32), f.view(np.int32)), name
        out.update(enc)
        out[name + "_attention_factor"] = np.float64(rows[0][1])
    np.savez_compressed(os.path.join(HERE, "rope_len_inv_freq.npz"), **out)
    print("wrote", sorted(out))


if __name__ == "__main__":
    torch.set_num_threads(1)
    main()
