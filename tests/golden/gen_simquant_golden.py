#!/usr/bin/env python
"""Generate tests/golden/simquant_*.npz by importing the REFERENCE's own simulated-quant functions
(the reference's quant/kvquant/simquant_module_quantizer.py: get_outliers, get_outliers_dynamic,
quant_fn_nuq_recon, round_to_nearest_pole_sim) on CPU.  Needs a reference checkout
(oracle/build_ref.py: REF_ROOT); the produced fixtures are committed.

    python tests/golden/gen_simquant_golden.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))), "oracle"))
from build_ref import REF_ROOT  # noqa: E402
sys.path.insert(0, os.path.join(REF_ROOT, "quant"))

from kvquant.simquant_module_quantizer import (  # noqa: E402  (reference code, imported not copied)
    get_outliers, get_outliers_dynamic, quant_fn_nuq_recon, round_to_nearest_pole_sim)
from kvquant_b200 import synth  # noqa: E402


def main():
    torch.manual_seed(0)
    spec = synth.SynthSpec(32, 128, seed=0)
    T = 8
    for bits in (4, 3, 2):
        cal = synth.calibrate(spec, bits, calib_tokens=512, seed=7)
        k = spec.k_tokens(T, seed=100 + bits)
        v = spec.v_tokens(T, seed=200 + bits)
        up, lo, kc = cal["k"]
        vc = cal["v"][2]
        kt = torch.from_numpy(k)
        vt = torch.from_numpy(v)
        upt, lot = torch.from_numpy(up), torch.from_numpy(lo)
        out = {"bits": bits, "k": k, "v": v, "k_upper": up, "k_lower": lo,
               "k_cent": kc[0], "v_cent": vc[0]}
        # --- K: static per-channel thresholds (channel=0 broadcast over tokens), capped and uncapped
        for cap in (-1, 21):
            for ff in (-1, 2):
                m = get_outliers(kt, channel=0, outlier_threshold_upper=upt, outlier_threshold_lower=lot,
                                 cap_outliers=cap, first_few_fp16=ff)
                r = quant_fn_nuq_recon(kt, bits=bits, qchannel=0, dynamicquantization=False, include_sparse=True,
                                       outlier_mask=m, maxval=upt, minval=lot, lut=kc, first_few_fp16=ff)
                tag = "k_cap%d_ff%d" % (cap, ff)
                out[tag + "_mask"] = m.numpy()
                out[tag + "_recon"] = r.numpy()
        # --- K with Q-Norm
        m = get_outliers(kt, channel=0, outlier_threshold_upper=upt, outlier_threshold_lower=lot, cap_outliers=21)
        r = quant_fn_nuq_recon(kt, bits=bits, qchannel=0, include_sparse=True, outlier_mask=m, maxval=upt,
                               minval=lot, lut=kc, norm=True, normscale=torch.tensor(1.0625),
                               normoffset=torch.tensor(-0.015625))
        out["k_norm_recon"] = r.numpy()
        # --- V: dynamic per-token
        for ff in (-1, 2):
            m = get_outliers_dynamic(vt, channel=-1, thresh=0.99, first_few_fp16=ff)
            r = quant_fn_nuq_recon(vt, bits=bits, qchannel=-1, dynamicquantization=True, include_sparse=True,
                                   outlier_mask=m, lut=vc, first_few_fp16=ff)
            out["v_dyn_ff%d_mask" % ff] = m.numpy()
            out["v_dyn_ff%d_recon" % ff] = r.numpy()
        # dense-only dynamic V
        r = quant_fn_nuq_recon(vt, bits=bits, qchannel=-1, dynamicquantization=True, include_sparse=False, lut=vc)
        out["v_dense_recon"] = r.numpy()
        # round_to_nearest_pole_sim on a small vector incl. exact ties
        w = torch.tensor([-2.0, -0.5, 0.0, 0.25, 0.5, 0.75, 3.0], dtype=torch.float32)
        poles = torch.tensor([0.0, 0.5, -1.0, 1.0], dtype=torch.float32)
        out["pole_w"] = w.numpy()
        out["pole_p"] = poles.numpy()
        out["pole_out"] = round_to_nearest_pole_sim(w, poles).numpy()
        path = os.path.join(HERE, "simquant_b%d.npz" % bits)
        np.savez_compressed(path, **out)
        print("wrote", path, os.path.getsize(path))


if __name__ == "__main__":
    main()
