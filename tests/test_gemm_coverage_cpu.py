"""Coverage guard of the GEMM kernel matrix (no GPU): every gemm_i8_kernel<MODE, W4> instantiation that engine.cu's
launch_gemm can launch has a row in tests/test_gemm_matrix_gpu.py's INSTANTIATIONS, and every row names a case that
expects exactly that instantiation (or says why no descriptor reaches it).  A mode added to launch_gemm without a test
fails here on a machine with no GPU."""
import os
import re

from tests import test_gemm_matrix_gpu as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "q-diffusion_b200", "csrc")


def _epi_bits():
    src = open(os.path.join(CSRC, "gemm_i8.cuh")).read()
    return {k: int(v) for k, v in re.findall(r"constexpr int (EPI_[A-Z0-9_]+)\s*=\s*(\d+);", src)}


def _launched_pairs():
    """(MODE, W4) of every launch_gemm_mode<MODE> (both W4 forms: it dispatches on the run-time flag) and
    launch_gemm_mode_w<MODE, W4> in the body of launch_gemm."""
    src = open(os.path.join(CSRC, "engine.cu")).read()
    body = re.search(r"\nint launch_gemm\(const GemmPlan& pl, cudaStream_t s\) \{\n(.*?)\n\}\n", src, re.S)
    assert body, "launch_gemm not found in engine.cu"
    bits = _epi_bits()

    def mode(expr):
        expr = expr.strip()
        if re.fullmatch(r"-?\d+", expr):
            return int(expr)
        v = 0
        for name in expr.split("|"):
            v |= bits[name.strip()]
        return v

    pairs = set()
    for wrapper, args in re.findall(r"(launch_gemm_mode(?:_w)?)<([^<>]+)>\(", body.group(1)):
        if wrapper == "launch_gemm_mode":
            pairs |= {(mode(args), False), (mode(args), True)}
        else:
            expr, w4 = args.rsplit(",", 1)
            pairs.add((mode(expr), w4.strip() == "true"))
    return pairs


def test_mode_bits_match_the_kernel():
    bits = _epi_bits()
    want = dict(EPI_CORR=G.CORR, EPI_ROWVEC=G.ROWVEC, EPI_RESIDUAL=G.RES, EPI_OUT_F32=G.F32, EPI_OUT_Q=G.Q,
                EPI_GEGLU=G.GEGLU, EPI_TRANS=G.TRANS, EPI_CONV=G.CONV, EPI_RESTMA=G.RESTMA, EPI_BF16=G.BF16,
                EPI_SPLITK=G.SPLITK)
    assert bits == want, (bits, want)


def test_every_instantiation_has_a_row():
    launched = _launched_pairs()
    assert len(launched) >= 60, len(launched)
    assert set(G.INSTANTIATIONS) == launched, (
        f"missing rows: {sorted(launched - set(G.INSTANTIATIONS))}; rows without an instantiation: "
        f"{sorted(set(G.INSTANTIATIONS) - launched)}")


def test_every_row_names_a_case_that_expects_it():
    for key, row in G.INSTANTIATIONS.items():
        if row.startswith("unreachable: "):
            assert len(row) > len("unreachable: ") + 10, key
            continue
        assert row in G.CASES, (key, row)
        expect = G.CASES[row]["expect"]
        assert (expect == "splitk" and key == (G.SPLITK, False)) or expect == key, (key, row, expect)


def test_every_case_expects_an_instantiation():
    for cid, c in G.CASES.items():
        assert c["expect"] == "splitk" or c["expect"] in G.INSTANTIATIONS, (cid, c["expect"])
        assert not str(G.INSTANTIATIONS.get(c["expect"], "")).startswith("unreachable"), cid
        if c["twin"] is not None:
            assert c["twin"] in G.INSTANTIATIONS, cid


def test_every_n_tile_runs_for_both_signednesses():
    """The fp32 int8 matrix runs each of the eight N tiles (gemm_dispatch_bn) with u8 and with s8 codes; split-K covers
    the wide tiles with 0-4 full blocks and every tail."""
    seen = {(c["bn"], c["sym"]) for cid, c in G.CASES.items() if cid.startswith("f32-")}
    assert {(bn, sym) for bn in G.BNS for sym in (False, True)} <= seen
    wide = {min(c["N"], 256) for cid, c in G.CASES.items() if cid.startswith("splitk-")}
    assert {(n // 64, n % 64) for n in wide} >= {(0, 48), (1, 32), (2, 16), (2, 48), (3, 32), (3, 48), (4, 0)}
