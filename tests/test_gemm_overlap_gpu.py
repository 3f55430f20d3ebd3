"""The overlapped INT8 GEMM schedule over many work items per CTA.

Every gemm_i8_kernel instantiation that runs its epilogue on dedicated epilogue warps (csrc/gemm_i8.cuh gemm_overlap)
hands one accumulator tile between the consumer warpgroups and the epilogue warps through two mbarriers, acc_full and
acc_empty, whose phases advance once per work item.  The cases of tests/test_gemm_matrix_gpu.py give a CTA at most two
work items; here every case has at least four per CTA (more than 4 x 132 tiles), so both barriers wrap their phase
parity more than once.  Short-K cases (one k-block) have epilogues longer than the main loop, so the consumers wait on
acc_empty; long-K cases (24 k-blocks and more) have the epilogue warps waiting on acc_full.  The N tiles 16, 48, 112 and
128 are forced with bn_hint.  Inputs, the exact integer oracle, the tolerances and the profiler check of which
instantiation ran are those of test_gemm_matrix_gpu.py."""
import pytest

from tests import test_gemm_matrix_gpu as G

pytestmark = pytest.mark.gpu

CORR, ROWVEC, RES, F32, Q, GEGLU, TRANS, CONV, RESTMA = G.CORR, G.ROWVEC, G.RES, G.F32, G.Q, G.GEGLU, G.TRANS, G.CONV, G.RESTMA
TILES = 530       # > 4 work items per CTA on up to 132 SMs (asserted against the device)
K1, K24 = 96, 3072          # plain GEMM reduction lengths: 1 and 24 k-blocks of 128
CONV_C1, CONV_C27 = 32, 320  # 3x3 convs: 9 x 1 and 9 x 3 k-blocks


def _tiles_m(N, bn):
    return -(-TILES // -(-N // bn))


def _sign(sym):
    return "s8" if sym else "u8"


OVL = []


def _add(cid, expect, **spec):
    cid = "ovl-" + cid
    G._add(cid, (expect, False), **spec)
    OVL.append(cid)


def _plain(cid, bits, sym, N, bn, C, **kw):
    _add(cid, bits | (0 if sym else CORR), M=128 * _tiles_m(N, bn) - 45, N=N, C=C, sym=sym, bn=bn, **kw)


# fp32 outputs: plain / per-image vector (short K), residual through registers (long K only: the ring takes <= 5 k-blocks)
# and through the TMA ring (short K), GroupNorm slab statistics
_plain("f32-s8-k1-bn128", F32, True, 256, 128, K1)
_plain("f32-u8-k1-bn16-gn", F32, False, 80, 16, K1, gn=True)
_plain("f32-u8-k24-bn16", F32, False, 64, 16, K24)
_plain("f32-rowvec-s8-k1-bn48", F32 | ROWVEC, True, 96, 48, K1, rowvec=True)
_plain("f32-rowvec-u8-k1-bn112", F32 | ROWVEC, False, 224, 112, K1, rowvec=True)
_plain("f32-res-s8-k24-bn16", F32 | RES, True, 64, 16, K24, res="alias")
_plain("f32-res-u8-k24-bn48-gn", F32 | RES, False, 48, 48, K24, res="sep", gn=True)
_plain("f32-restma-s8-k1-bn128", F32 | RES | RESTMA, True, 256, 128, K1, res="alias")
_plain("f32-restma-u8-k1-bn48", F32 | RES | RESTMA, False, 96, 48, K1, res="sep")
# requantised codes: plain (short and long K), residual through registers (long K) and through the ring (short K)
_plain("q-s8-k1-bn112", Q, True, 224, 112, K1, out_f=False, out_q="row")
_plain("q-u8-k24-bn16", Q, False, 64, 16, K24, out_f=False, out_q="row")
_plain("qres-s8-k24-bn16", Q | RES, True, 48, 16, K24, out_f=False, out_q="row", res="sep")
_plain("qres-u8-k24-bn16", Q | RES, False, 64, 16, K24, out_f=False, out_q="row", res="sep")
_plain("qrestma-s8-k1-bn48", Q | RES | RESTMA, True, 96, 48, K1, out_f=False, out_q="row", res="sep")
_plain("qrestma-u8-k1-bn128", Q | RES | RESTMA, False, 256, 128, K1, out_f=False, out_q="row", res="sep")
# GEGLU (N tiles are multiples of 32) and the V^T output (T = 64 tokens per image)
_plain("geglu-s8-k1-bn128", GEGLU | Q, True, 320, 128, K1, geglu=True, out_f=False, out_q="row")
_plain("geglu-u8-k24-bn32", GEGLU | Q, False, 64, 32, K24, geglu=True, out_f=False, out_q="row")
for sym, N, bn, C in ((True, 112, 16, K1), (False, 96, 48, K24)):
    _add(f"trans-{_sign(sym)}-k{C // 128 or 1}-bn{bn}", TRANS | Q | (0 if sym else CORR), M=128 * _tiles_m(N, bn), T=64,
         N=N, C=C, sym=sym, bn=bn, out_f=False, out_q="trans", ldq_pad=16)
# 3x3 convs, one 8 x 16 image per tile: border-class correction, per-image vector, residual, codes; 9 and 27 k-blocks
for epi, bits, kw in (("plain", F32, {}), ("rowvec", F32 | ROWVEC, dict(rowvec=True)), ("res", F32 | RES, dict(res="sep")),
                      ("q", Q, dict(out_f=False, out_q="row"))):
    for sym in (True, False):
        long_k = sym == (epi in ("plain", "q"))
        N, bn = (64, 16) if long_k else (96, 48)
        C = CONV_C27 if long_k else CONV_C1
        if epi == "plain" and not sym:
            kw = dict(gn=True)
        _add(f"conv-{epi}-{_sign(sym)}-k{9 * -(-C // 128)}-bn{bn}", bits | CONV | (0 if sym else CORR), taps=9,
             bhw=(_tiles_m(N, bn), 8, 16), N=N, C=C, sym=sym, bn=bn, **kw)


@pytest.mark.parametrize("cid", OVL)
def test_overlap(cuda, cid):
    s = G.CASES[cid]
    M = s["bhw"][0] * 128 if s["taps"] == 9 else s["M"]
    tiles = -(-M // 128) * -(-s["N"] // s["bn"])
    assert tiles >= 4 * G._sms(), (cid, tiles, G._sms())
    G.check_all(G.run_case(cuda, cid))


def test_covers_every_overlapped_instantiation():
    """Every instantiation on the overlapped schedule (int8, specialised epilogue, s8 weights) has a case here."""
    seen = {G.CASES[c]["expect"] for c in OVL}
    want = {k for k in G.INSTANTIATIONS if k[0] >= 0 and not k[1] and not k[0] & (G.BF16 | G.SPLITK)}
    assert seen == want, sorted(want - seen)
