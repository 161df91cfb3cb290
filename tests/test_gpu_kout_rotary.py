"""GPU: the rotary factors of the K outlier pass at long contexts.

Past 64K positions the outlier pass evaluates cos / sin of theta_j * pos itself, with theta_j staged once per CTA,
and reads only the arguments past cosf / sinf's fast argument reduction (CUDART_TRIG_PLOSS_F = 105615) from the rope
table.  These tests pin that every factor it uses is the rope table's, bit for bit:
  * exhaustively, for all 64 rotary rows and every position below 2^20 + 64 (one outlier per (token, head) through the
    legacy K op, whose dense part is zero);
  * on oracle caches placed at positions that straddle 105615 / theta_j for rows 0, 1 and 15, 64K and the end of a
    fresh rope table: equal bit for bit to the gather form (KVQ_KOUT_DIRECT_NPOS forces it, in a subprocess: the
    switch is read once per process).
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from _util import O, oracle_cache, spec

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HERE = os.path.dirname(os.path.abspath(__file__))
THETA = 10000.0
TRIG_FAST_MAX = 105615.0


def _row_limit(j):
    """first position whose argument theta_j * pos passes the fast reduction (float32 theta_j, as the kernels)."""
    th = np.float32(THETA) ** np.float32(-2.0 * j / 128.0)
    return int(TRIG_FAST_MAX / float(th)) + 1


def test_rotary_factors_equal_rope_table_exhaustive():
    from kvquant_b200 import quant_cuda as qc
    H, bits, L = 64, 2, (1 << 20) + 64
    W = 128 * bits // 32
    cache = torch.zeros((H, W, L), dtype=torch.int32, device=DEV)
    lut = torch.zeros((H, 128, 1 << bits), dtype=torch.float32, device=DEV)
    # token t: head h holds one outlier of value 1 on channel h (rotary row h, first half)
    idx = (torch.arange(H, dtype=torch.int32, device=DEV) * 129).expand(L, H).contiguous()
    val = torch.ones((L, H), dtype=torch.float32, device=DEV)
    rope, npos = qc.rope_table(torch.device(DEV), THETA, L)
    rope = rope[:, :L]
    for k, want in ((0, rope[..., 0]), (1, rope[..., 1])):   # q on channel h -> cos; on channel h + 64 -> sin
        q = torch.zeros((1, H, 128), dtype=torch.float32, device=DEV)
        q[0, torch.arange(H), torch.arange(H) + 64 * k] = 1.0
        mul = torch.zeros((1, H, L), dtype=torch.float32, device=DEV)
        qc._k_matvec(bits, q, cache, mul, lut, L, val, idx, THETA, 0)
        got = mul[0]
        bad = (got.view(torch.int32) != want.contiguous().view(torch.int32)) & ~((got == 0) & (want == 0))
        n_bad = int(bad.sum())
        assert n_bad == 0, (k, n_bad, torch.nonzero(bad)[:8].tolist())
        del mul
    torch.cuda.synchronize()


BITS = (4, 3, 2)
L_CASE = 611
# (name, pos_offset): the L_CASE positions [off, off + L_CASE) straddle the named point
OFFSETS = (("row0_limit", _row_limit(0) - L_CASE // 2), ("row1_limit", _row_limit(1) - L_CASE // 2),
           ("64K", 65536 - L_CASE // 2), ("row15_limit", _row_limit(15) - L_CASE // 2))
TABLE_END = 2 * 1024 * 1024 - L_CASE   # last position = the last entry of a table built for exactly 2^21 positions


def _k_scores(bits, off):
    from kvquant_b200 import quant_cuda as qc
    import test_gpu_parity as P
    c, _, _ = oracle_cache(bits, L_CASE)
    d = P.device_cache(c)
    q = O.rope_rotate_q(spec().q_vec(5), L_CASE + off, THETA)
    mul = torch.zeros((1, c.H, L_CASE), dtype=torch.float32, device=DEV)
    qc._k_matvec(bits, P.cu(q[None]), d["kcache"], mul, d["klut"], L_CASE, d["k_out"], d["k_idx"], THETA, off)
    return c, q, mul.cpu().numpy()[0]


CHILD = r"""
import sys
sys.path.insert(0, %r)
import numpy as np
import test_gpu_kout_rotary as T
out = {}
for bits in T.BITS:
    for name, off in T.OFFSETS + (("table_end", T.TABLE_END),):
        out["%%d_%%s" %% (bits, name)] = T._k_scores(bits, off)[2]
np.savez(sys.argv[1], **out)
print("CHILD_OK")
""" % HERE


@pytest.fixture(scope="module")
def gather_form(tmp_path_factory):
    """K scores of every case with every outlier factor gathered from the rope table."""
    path = str(tmp_path_factory.mktemp("kout") / "gather.npz")
    env = dict(os.environ, KVQ_KOUT_DIRECT_NPOS=str(1 << 40))
    r = subprocess.run([sys.executable, "-c", CHILD, path], env=env, capture_output=True, text=True, timeout=900,
                       cwd=HERE)
    assert r.returncode == 0 and "CHILD_OK" in r.stdout, (r.stdout[-2000:], r.stderr[-2000:])
    return dict(np.load(path))


@pytest.mark.parametrize("bits", BITS)
@pytest.mark.parametrize("name,off", OFFSETS + (("table_end", TABLE_END),))
def test_long_position_outliers_match_gather_form(bits, name, off, gather_form):
    from kvquant_b200 import quant_cuda as qc
    if name == "table_end":   # the last position is the table's last entry unless a larger table was built before
        qc.rope_table(torch.device(DEV), THETA, off + L_CASE)
    c, _, got = _k_scores(bits, off)
    rows = np.unique(c.k_idx[:L_CASE][c.k_out[:L_CASE] != 0] & 63)
    assert {0, 1, 15} <= set(rows.tolist())
    want = gather_form["%d_%s" % (bits, name)]
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), int((got != want).sum())
