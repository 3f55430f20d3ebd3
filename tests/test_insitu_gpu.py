"""Deterministic per-op parity gate (VERDICT r1 item 1b): every recorded engine op of every golden UNet - and of the
full-size CIFAR-10 / LSUN-church (W8A8) / SD v1-4 UNets - is replayed on its own and checked against the CPU oracle
evaluated on the engine's inputs of that op (tests/insitu.py states the tolerances: bit-exact for integer ops, <= 1
code at < 2e-3 of positions behind fp32 arithmetic), and the folded integer weights of every QuantModule must equal
the oracle's fake-quant weights bit for bit.  The per-op report goes to $QDIFF_REPORT_DIR (default
<tmp>/qdiff_reports) and, summarised, to stdout; tools/parity_report.py assembles a parity report from it."""
import json
import os
import tempfile

import pytest
import torch

from tests import insitu
from tests.test_oracle_golden import CASES, ORACLE_ONLY, load_case
from tests.test_unet_gpu import build_qnn

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _dump(name, rep, extra=None):
    out = os.environ.get("QDIFF_REPORT_DIR") or os.path.join(tempfile.gettempdir(), "qdiff_reports")      # diagnostic report, outside the tree
    try:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, f"insitu_{name}.json"), "w") as f:
            json.dump(dict(case=name, rows=rep.rows, extra=extra or {}), f)
    except OSError:
        pass


def _run(name, qnn, x, t, ctx, cuda, device="cpu"):
    c = ctx.to(cuda) if ctx is not None else None
    prog = qnn.program(x.to(cuda), c)
    rep = insitu.verify_program(prog, x, t, ctx, device=device)
    kinds = {s["kind"] for s in prog.op_specs}
    print(f"\n[{name}] in-situ per-op parity: {prog.nops} ops, kinds {sorted(kinds)}\n{rep.summary()}")
    txt = rep.text()
    if txt:
        print(txt[:6000])
    return prog, rep


@pytest.mark.parametrize("name", CASES + ORACLE_ONLY)      # ORACLE_ONLY: the weight-only fixture (BASELINE configs[0])
def test_every_op_matches_oracle_on_golden_unets(cuda, name):
    g = load_case(name)
    qnn = build_qnn(g, cuda)
    qnn.record_op_specs = True
    n, bad = insitu.verify_folds(qnn, g, cuda)
    prog, rep = _run(name, qnn, g["x"], g["t"], g["context"], cuda)
    _dump(name, rep, dict(folds=n, folds_bad=bad, nops=prog.nops))
    assert n > 0 and bad == 0, f"{bad}/{n} folded weight tensors differ from the oracle's fake-quant weights"
    assert "unspecified" not in {s["kind"] for s in prog.op_specs}
    fails = rep.failures()
    assert not fails, "\n".join(f"op {r['idx']} {r['kind']} {r['label']} {r['what']} bad={r['nbad']}/{r['n']} max={r['maxdiff']}"
                                for r in fails[:20])
    # every QuantModule of the model is covered by at least one checked GEMM op
    covered = {s["key"] for s in prog.op_specs if s["kind"] in ("gemm", "gemm_wo")}
    modules = {k for k, m in qnn.model.named_modules() if type(m).__name__ == "QuantModule"}
    assert modules <= covered, sorted(modules - covered)[:10]


@pytest.mark.parametrize("name,batch", [("cifar10", 2), ("lsun_church", 1), ("sd_v1", 1)])
def test_every_op_matches_oracle_fullsize(cuda, name, batch):
    """BASELINE.json UNets at full size (cfg 2 CIFAR-10 W4A8 split, cfg 5 LSUN-church W8A8, cfg 4 SD v1-4 W4A8 sm16); the
    oracle runs on the device."""
    from qdiff_b200 import synth
    qnn, ckpt = synth.build_qnn(name)
    qnn.record_op_specs = True
    x, t, ctx = synth.calib_inputs(name, batch=batch, seed=4242)
    prog, rep = _run(f"{name}_full", qnn, x, t, ctx, cuda, device=cuda)        # the float64 oracle on the device
    _dump(f"{name}_full", rep, dict(nops=prog.nops))
    fails = rep.failures()
    assert not fails, "\n".join(f"op {r['idx']} {r['kind']} {r['label']} {r['what']} bad={r['nbad']}/{r['n']} max={r['maxdiff']}"
                                for r in fails[:20])
