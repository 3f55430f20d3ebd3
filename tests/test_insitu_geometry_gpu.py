"""The per-op in-situ gate (tests/insitu.py, tolerances unchanged) at the inputs the golden fixtures never reach:

  * latents the implicit-GEMM conv does not tile (Builder.implicit_conv_ok false at every level, so every stride-1 3x3 conv
    is an explicit patch gather + plain GEMM whose 128-row tiles straddle images): 24x24 (levels 24, 12) and 12x12
    (levels 12, 6; the 6x6 level has H*W < 128 and does not divide 128), at batches 3 and 1, timesteps 0, 1, 999 and a
    fractional DPM-Solver model time, both timestep-embedding modes (LDM and DDIM families), every golden UNet;
  * the weight-only (bfloat16-plane) state at 24x24;
  * the classifier-free-guidance program (program(..., cfg_dedup=True)) of the conditional fixture, at 16x16 guided
    batch 8, where the GroupNorm slab sums are copied with the activations, at 24x24 guided batch 8, and at 12x12 guided
    batch 3, where half the batch is 432 rows and the slab copy is skipped;
  * full size: SD v1-4 guided at 96x96 latents, one image (UNet batch 2: self-attention at T = 9216 / 2304 / 576 / 144,
    the patch-gather conv at every level), and at 64x64, batch 8 (UNet batch 16: the benchmark's shape), with the float64
    oracle on the device;
  * the first DPM-Solver call on the CIFAR-style fixture (x_T at t = 999, the seeds of
    test_samplers_ext_gpu.py::test_dpm_solver_singlestep_quantised_matches_oracle) and its second, fractional call.

Negative controls perturb the oracle's copy of a spec (verify_program's alter) and must make the gate fail: a rowvec
shifted by one image in a patch-gather conv, a dropped slab-sum copy, a timestep off by one at t = 999.
Each case prints its op count, its op kinds and the per-kind summary, and dumps its rows like test_insitu_gpu.py."""
import time

import pytest
import torch

from tests import insitu
from tests.test_insitu_gpu import _dump
from tests.test_oracle_golden import CASES, ORACLE_ONLY, load_case
from tests.test_unet_gpu import build_qnn

pytestmark = pytest.mark.gpu

FRAC = 832.3333          # a fractional DPM-Solver model time (t - 1/N) * 1000
TIMES = {3: [0.0, 999.0, FRAC], 1: [1.0], 8: [999.0, 0.0, 1.0, FRAC, 500.0, 1.0, 999.0, 250.5]}
GEOMETRY = [(24, 3), (12, 1)]       # (latent size, batch): the patch-gather conv at every level of the two-level fixtures


def _inputs(g, size, batch, seed, guided=False):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(batch, g["x"].shape[1], size, size, generator=gen)
    t = torch.tensor(TIMES[batch], dtype=torch.float32)
    ctx = None
    if g["context"] is not None:
        ctx = torch.randn((2 if guided else 1) * batch, *g["context"].shape[1:], generator=gen)
    return x, t, ctx


def _gate(name, qnn, x, t, ctx, cuda, guided=False, device="cpu", alter=None):
    """Compile the program for these inputs, run the per-op gate on it and print what it covered."""
    t0 = time.time()
    prog = qnn.program(x.to(cuda), ctx.to(cuda) if ctx is not None else None, cfg_dedup=guided)
    rep = insitu.verify_program(prog, x, t, ctx, alter=alter, device=device)
    if alter is None:
        kinds = sorted({s["kind"] for s in prog.op_specs})
        print(f"\n[{name}] {prog.nops} ops in {time.time() - t0:.1f} s, kinds {kinds}\n{rep.summary()}")
        txt = rep.text()
        if txt:
            print(txt[:6000])
        _dump(name, rep, dict(nops=prog.nops))
    return prog, rep


def _assert_clean(prog, rep):
    assert "unspecified" not in {s["kind"] for s in prog.op_specs}
    fails = rep.failures()
    assert not fails, "\n".join(f"op {r['idx']} {r['kind']} {r['label']} {r['what']} bad={r['nbad']}/{r['n']} max={r['maxdiff']}"
                                for r in fails[:20])


def _labels(prog, label):
    return [i for i, n in enumerate(prog.op_names) if n == label]


# ------------------------------------------------------------------------------------------------ golden UNets
@pytest.mark.parametrize("size,batch", GEOMETRY)
@pytest.mark.parametrize("name", CASES + ORACLE_ONLY)
def test_every_op_at_non_tiling_latents(cuda, name, size, batch):
    g = load_case(name)
    qnn = build_qnn(g, cuda)
    qnn.record_op_specs = True
    if (size, batch) == GEOMETRY[0]:
        n, bad = insitu.verify_folds(qnn, g, cuda)
        assert n > 0 and bad == 0, f"{bad}/{n} folded weight tensors differ from the oracle's fake-quant weights"
    x, t, ctx = _inputs(g, size, batch, seed=size + batch)
    prog, rep = _gate(f"{name}_{size}x{size}_b{batch}", qnn, x, t, ctx, cuda)
    _assert_clean(prog, rep)
    gathers = [s for s in prog.op_specs if s["kind"] in ("im2col", "im2col_bytes") and s["stride"] == 1]
    assert {(s["H"], s["W"]) for s in gathers} == {(size, size), (size // 2, size // 2)}


@pytest.mark.parametrize("name", ["sd_tiny_w4_weightonly", "ldm_updown_w8_weightonly"])
def test_weight_only_state_at_non_tiling_latents(cuda, name):
    g = load_case(name)
    qnn = build_qnn(g, cuda)
    qnn.set_quant_state(True, False)
    qnn.record_op_specs = True
    x, t, ctx = _inputs(g, 24, 3, seed=7)
    prog, rep = _gate(f"{name}_24x24_b3_weight_only", qnn, x, t, ctx, cuda)
    _assert_clean(prog, rep)
    assert {"im2col_bytes", "gemm_wo"} <= {s["kind"] for s in prog.op_specs}


# ------------------------------------------------------------------------------------------------ guided programs
@pytest.mark.parametrize("size,batch,slab_copy", [(16, 8, True), (24, 8, True), (12, 3, False)])
def test_guided_program(cuda, size, batch, slab_copy):
    g = load_case("sd_tiny_w4a8_sm16")
    qnn = build_qnn(g, cuda)
    qnn.record_op_specs = True
    x, t, ctx = _inputs(g, size, batch, seed=100 + size, guided=True)
    prog, rep = _gate(f"sd_tiny_w4a8_sm16_guided_{size}x{size}_b{batch}", qnn, x, t, ctx, cuda, guided=True)
    _assert_clean(prog, rep)
    assert _labels(prog, "cfg.dup")
    assert bool(_labels(prog, "cfg.dup.slabs")) == slab_copy


# ------------------------------------------------------------------------------------------------ full size
@pytest.mark.parametrize("size,batch", [(96, 1), (64, 8)])
def test_sd_v1_guided_fullsize(cuda, size, batch):
    """SD v1-4 (seeded weights, BASELINE cfg 4 W4A8 sm16) through forward_cfg's program; the oracle runs on the device."""
    from qdiff_b200 import synth
    qnn, _ = synth.build_qnn("sd_v1")
    qnn.record_op_specs = True
    gen = torch.Generator().manual_seed(4243)
    x = torch.randn(batch, 4, size, size, generator=gen)
    t = torch.tensor(TIMES[batch], dtype=torch.float32)
    ctx = torch.randn(2 * batch, 77, 768, generator=gen)
    prog, rep = _gate(f"sd_v1_guided_{size}x{size}_b{batch}", qnn, x, t, ctx, cuda, guided=True, device=cuda)
    _assert_clean(prog, rep)
    assert _labels(prog, "cfg.dup.slabs")
    if size == 96:
        Ts = {s["Tq"] for s in prog.op_specs if s["kind"] == "attention" and s["Tq"] == s["Tk"]}
        assert Ts == {9216, 2304, 576, 144}, Ts


# ------------------------------------------------------------------------------------------------ DPM-Solver call 0
class _Stop(Exception):
    pass


def _dpm_calls(g, x, steps, n):
    """The first n UNet calls (x, t) of the oracle's singlestep DPM-Solver loop on x."""
    from oracle import sampler_ext_oracle as SX
    from tests.test_samplers_ext_gpu import _ddim_betas
    from tests.test_samplers_gpu import RecordingOracle
    lo = RecordingOracle(g)

    def model(xx, tt):
        if len(lo.calls) == n:
            raise _Stop
        return lo(xx, tt)
    try:
        SX.dpm_solver_singlestep(model, x, _ddim_betas(), steps)
    except _Stop:
        pass
    return lo.calls


@pytest.mark.parametrize("steps", [6, 7])
def test_dpm_solver_first_calls(cuda, steps):
    """x_T at t = 999 (call 0) and the fractional call 1, on the inputs of test_dpm_solver_singlestep_quantised_matches_oracle.
    Also prints the engine's eps MSE from the oracle next to the oracle's fp32-vs-fp64 band at t = 999 and nearby t."""
    from tests.test_samplers_gpu import RecordingOracle
    g = load_case("ddim_w4a8_split")
    qnn = build_qnn(g, cuda)
    qnn.record_op_specs = True
    x = torch.randn(2, *g["x"].shape[1:], generator=torch.Generator().manual_seed(62 + steps))
    calls = _dpm_calls(g, x, steps, 2)
    assert float(calls[0][1][0]) == 999.0 and float(calls[1][1][0]) != round(float(calls[1][1][0]))
    for k, (xx, tt, _, _) in enumerate(calls):
        prog, rep = _gate(f"ddim_w4a8_split_dpm{steps}_call{k}_t{float(tt[0]):.2f}", qnn, xx, tt, None, cuda)
        _assert_clean(prog, rep)
    lo, hi = RecordingOracle(g, record=False), RecordingOracle(g, torch.float64, record=False)
    print(f"\n[dpm{steps} x_T] eps MSE, engine vs fp32 oracle, and the oracle's fp32 vs fp64 band:")
    for tv in (999, 990, 900, 500, 10):
        tt = torch.full((2,), float(tv))
        e32 = lo(x, tt)
        e_eng = qnn(x.to(cuda), tt.to(cuda)).cpu()
        band = float(((hi(x.double(), tt) - e32.double()) ** 2).mean())
        print(f"   t={tv:4d}  engine {float(((e_eng.double() - e32.double()) ** 2).mean()):.3e}  band {band:.3e}")


# ------------------------------------------------------------------------------------------------ negative controls
def _failing_ops(rep):
    return {r["idx"] for r in rep.failures()}


def _altering(pred, change):
    """alter hook: change(spec) for the specs pred selects; records which ops it touched (by spec identity)."""
    hit = []

    def f(s):
        if not pred(s):
            return s
        hit.append(id(s))
        return change(s)
    return f, hit


def _touched(prog, hit):
    return {i for i, s in enumerate(prog.op_specs) if id(s) in hit}


@pytest.mark.parametrize("name", ["ddim_w4a8_split", "ldm_legacy_w4a8"])        # (the scale-shift fixtures have no rowvec)
def test_negative_rowvec_shifted_by_one_image_in_a_gather_conv(cuda, name):
    from qdiff_b200.graph import Act
    g = load_case(name)
    qnn = build_qnn(g, cuda)
    qnn.record_op_specs = True
    x, t, ctx = _inputs(g, 24, 3, seed=11)

    def shifted(s):
        rv = s["rowvec"]
        return dict(s, rowvec=Act(torch.roll(rv.logical(), 1, 0).contiguous(), rv.rows, rv.cols))
    alter, hit = _altering(lambda s: s["kind"] == "gemm" and s["rowvec"] is not None and s["taps"] == 1
                           and s["rows_per_batch"] % 128 != 0, shifted)
    prog, rep = _gate("neg", qnn, x, t, ctx, cuda, alter=alter)
    touched = _touched(prog, hit)
    assert touched and _failing_ops(rep) == touched


def test_negative_dropped_slab_sum_copy(cuda):
    g = load_case("sd_tiny_w4a8_sm16")
    qnn = build_qnn(g, cuda)
    qnn.record_op_specs = True
    x, t, ctx = _inputs(g, 16, 8, seed=116, guided=True)
    # the oracle reads the second half's slab sums from a copy of the table taken before the op: what they would hold
    # had the engine skipped the copy
    alter, hit = _altering(lambda s: s["kind"] == "cfg_dup" and "slabs" in s, lambda s: dict(s, slabs=s["slabs"].clone()))
    prog, rep = _gate("neg", qnn, x, t, ctx, cuda, guided=True, alter=alter)
    touched = _touched(prog, hit)
    assert touched and _failing_ops(rep) == touched


@pytest.mark.parametrize("name", ["ddim_w4a8_split", "ldm_legacy_w4a8"])
def test_negative_timestep_off_by_one_at_999(cuda, name):
    g = load_case(name)
    qnn = build_qnn(g, cuda)
    qnn.record_op_specs = True
    x = torch.randn(2, *g["x"].shape[1:], generator=torch.Generator().manual_seed(68))
    alter, hit = _altering(lambda s: s["kind"] == "timestep_emb", lambda s: dict(s, t=s["t"] - 1))
    prog, rep = _gate("neg", qnn, x, torch.full((2,), 999.0), None, cuda, alter=alter)
    touched = _touched(prog, hit)
    assert len(touched) == 1 and _failing_ops(rep) == touched
