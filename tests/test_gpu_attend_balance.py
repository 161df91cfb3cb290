"""GPU: the exact K kernel of the fused attend (k_ratio_kernel, kvq_kratio.cu) at lengths where a CTA's last round of
16-token columns has 1, 14 or 15 live columns.  The last round spreads its (column, head) units over all 15 consumer
warps; each score is still computed by one warp with the same instruction sequence, so:
  * the attend agrees with float64 at 2, 3 and 4 bits, MHA and GQA, dense and K+V-outlier caches;
  * on dense caches repeated calls are bit-identical, and a captured dynamic-length step replayed 16 times (the length
    crossing column and round boundaries) equals the same steps run eagerly, bit for bit;
  * the paged attend stays bit-identical to the contiguous batched attend.
A CTA's token range is the length over the CTAs of a head group rounded up to whole columns, so L = splits * 16 * n
gives every CTA exactly n columns."""
import pytest
import torch

import test_gpu_batch as TB
import test_gpu_gqa as G
import test_gpu_paged as PG

pytestmark = pytest.mark.gpu
DEV = G.DEV
COLS = (1, 14, 15, 16)    # columns per CTA: last round with 1 / 14 / 15 live columns, one or two rounds


def _splits(bits, Hq):
    """CTAs per head group: the SMs shared by ceil(Hq / heads-per-CTA) head groups (16 heads at 4 bits, 32 below)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return sms // -(-Hq // (16 if bits == 4 else 32))


def _length(bits, Hq, cols):
    return _splits(bits, Hq) * 16 * cols


@pytest.mark.parametrize("mode", ["kv", "dense"])
@pytest.mark.parametrize("Hq,Hkv", [(8, 8), (32, 8)])
@pytest.mark.parametrize("bits", [4, 3, 2])
def test_attend_against_float64_at_partial_rounds(bits, Hq, Hkv, mode):
    lens = [_length(bits, Hq, c) for c in COLS]
    lens += [lens[-1] - 1, lens[-1] + 1]                 # the last CTA one token short / one CTA of a single token
    lc = G._cache(bits, Hq, Hkv, mode, Lmax=(max(lens) + 7) // 4 * 4)
    lc.append_chunk(*G._tokens(lc, max(lens), seed=bits * 10 + Hq))
    q = G._query(Hq, bits)
    for L in lens:
        lc.len = L
        out = G._attend(lc, q)
        G._check(out, G._oracle_gqa(lc, q), "L=%d" % L)
        if mode == "dense":
            again = G._attend(lc, q)
            assert torch.equal(out[0], again[0]) and torch.equal(out[1], again[1]), L


@pytest.mark.parametrize("Hq,Hkv", [(32, 32), (32, 8)])
def test_captured_dynamic_step_equals_eager_steps_bit_for_bit(Hq, Hkv):
    from kvquant_b200 import _lib
    bits = 3
    L0 = _length(bits, Hq, 15) - 8                       # replays cross a column and a round boundary
    lc = G._cache(bits, Hq, Hkv, "dense", Lmax=L0 + 64, n_sink=3)
    G._sinks(lc, 3, seed=1)
    k, v = G._tokens(lc, L0 + 16, seed=7)
    lc.append_chunk(k[:L0], v[:L0])
    q = G._query(Hq, 5)
    lc.len = L0
    len_dev = torch.full((1,), L0, dtype=torch.int64, device=DEV)
    kin, vin = torch.empty_like(k[0]), torch.empty_like(v[0])
    out = torch.empty((Hq, 128), device=DEV)
    lib = _lib.load()

    def step():
        lc.append_dyn(kin, vin, len_dev)
        lc.attend_dyn(q, len_dev, 1, out=out)
        _lib.check(lib.kvq_dec_counter_add(len_dev.data_ptr(), 1, torch.cuda.current_stream().cuda_stream))

    kin.copy_(k[L0]); vin.copy_(v[L0])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    len_dev.fill_(L0)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    len_dev.fill_(L0)
    got = []
    for i in range(16):
        kin.copy_(k[L0 + i]); vin.copy_(v[L0 + i])
        graph.replay()
        torch.cuda.synchronize()
        got.append(out.clone())
    assert int(len_dev.item()) == L0 + 16
    ref = G._cache(bits, Hq, Hkv, "dense", Lmax=L0 + 64, n_sink=3)
    ref.set_sinks(lc.sink_k, lc.sink_v)
    ref.append_chunk(k[:L0], v[:L0])
    for i in range(16):
        ref.append(k[L0 + i], v[L0 + i])
        assert torch.equal(G._attend(ref, q)[0], got[i]), i


@pytest.mark.parametrize("bits", [4, 3])
def test_paged_attend_equals_the_contiguous_batch_at_partial_rounds(bits):
    Hq, Hkv = 32, 8
    lens = (_length(bits, Hq, 1) + 5, 160 * 7, _length(bits, Hq, 14), 321)
    bc, pc, Lmax = PG._pair(bits, Hq, Hkv, lens, 160, "dense")
    q = TB._queries(pc, 6)
    out, lse = PG._pattend(pc, q, L_cap=Lmax)
    o1, l1 = TB._battend(bc, q, L_cap=Lmax)
    assert torch.equal(out, o1) and torch.equal(lse, l1)
    for b, L in enumerate(lens):
        G._check((out[b], lse[b]), G._oracle_gqa(bc.seq(b), q[b]), "seq %d (L=%d)" % (b, L))
