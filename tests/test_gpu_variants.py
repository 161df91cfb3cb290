"""GPU: the alternative outlier scatter kept behind an environment switch for A/B measurements (KVQ_KOUT_IMPL) and
the long-context form of the K outlier scatter (cos/sin evaluated directly instead of gathered from the rope table;
KVQ_KOUT_DIRECT_NPOS=0 forces it at test sizes) still agree with the oracle.  The switches are read once per process, so
each variant runs in a subprocess that executes the legacy K matvec parity check of test_gpu_parity.py."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))

SCRIPT = r"""
import sys
sys.path.insert(0, %r)
import test_gpu_parity as T
for bits, L, sparse in ((4, 1100, True), (3, 611, True), (2, 530, True), (3, 200, False)):
    T.test_k_matvec_matches_oracle(bits, L, sparse)
T.test_fused_attend_within_1e3_of_oracle_chain(4, 700, True, 3, "fp32")
T.test_fused_attend_within_1e3_of_oracle_chain(3, 611, True, 5, "fp16")
import os
if not os.environ.get("KVQ_KOUT_IMPL"):        # (the non-persistent outlier scatter takes its length from the host)
    T.test_device_resident_length_equals_host_length(4, 900, 0, "fp32")
    T.test_device_resident_length_equals_host_length(3, 611, 3, "fp16")
print("VARIANT_OK")
""" % HERE


@pytest.mark.parametrize("env", [{"KVQ_KOUT_IMPL": "table"}, {"KVQ_KOUT_DIRECT_NPOS": "0"}])
def test_variant_matches_oracle(env):
    e = dict(os.environ)
    e.update(env)
    r = subprocess.run([sys.executable, "-c", SCRIPT], env=e, capture_output=True, text=True, timeout=600, cwd=HERE)
    assert r.returncode == 0 and "VARIANT_OK" in r.stdout, (r.stdout[-2000:], r.stderr[-2000:])
