"""What a QuantModel carries between lowerings, checked without a GPU: the builders run against the recording library of
tools/dryrun_lowering.py and every lowered program is reduced to its op-stream digest (descriptors, buffer layout and
the contents of every buffer the ops read, folded weights included).

- Reload: a model that already lowered one checkpoint and then loads another must lower exactly what a model built
  fresh on the second checkpoint lowers.  The folded-weight cache (QuantModel._wcache) is keyed by op label, so a load
  that kept it would mix the old integer weights and steps with the new biases and quantizers.
- State toggling: set_quant_state keeps the folded weights on purpose; a toggle sequence must still lower, in each
  state, exactly what a fresh model put straight into that state lowers."""
import pytest
import torch

from tests.test_oracle_golden import load_case
from tests.test_unet_gpu import build_qnn
from tools.dryrun_lowering import digest, install_fake_lib

CPU = torch.device("cpu")


@pytest.fixture
def fake(monkeypatch):
    return install_fake_lib(monkeypatch.setattr)


def _lower(fake, qnn, g):
    """Digest of the program compile_unet would lower for the fixture's input shapes in the model's current state.
    The builders are driven directly (no Program object: its destructor would hand the fake engine handle to the
    real library once the fake is gone)."""
    from qdiff_b200 import graph
    states = {(m.use_weight_quant, m.use_act_quant) for m in qnn.model.modules() if type(m).__name__ == "QuantModule"}
    assert len(states) == 1
    cls = graph.Builder if states == {(True, True)} else graph.WeightOnlyBuilder
    x_shape = tuple(g["x"].shape)
    b = cls(qnn, CPU, x_shape[0])
    n0 = len(fake.descs)
    with torch.no_grad():
        if g["family"] == "ddim":
            b.lower_ddim(qnn.model, x_shape)
        else:
            b.lower_ldm(qnn.model, x_shape, tuple(g["context"].shape))
    b.flush()
    return digest(b, fake.descs[n0:])["digest"]


def _scaled(ckpt, s=1.25):
    """Another calibrated checkpoint of the same model: every weight, bias and weight step scaled by s (AdaRound alphas
    and activation quantizers kept)."""
    out = {}
    for k, v in ckpt.items():
        scale = k.endswith((".weight", ".bias")) or (".weight_quantizer" in k and k.endswith(".delta"))
        out[k] = v * s if scale else v.clone()
    return out


def _fresh(g, ckpt, state):
    qnn = build_qnn(dict(g, ckpt=ckpt), CPU)
    qnn.set_quant_state(*state)
    return qnn


@pytest.mark.parametrize("name,state", [
    ("ddim_w4a8_split", (True, True)),            # INT8 state: Builder._weights entries
    ("sd_tiny_w4a8_sm16", (True, True)),          # ... and the hoisted context K/V of an SD UNet
    ("ddim_w8_weightonly", (True, False)),        # weight-only state: integer codes as bfloat16 planes
    ("sd_tiny_w4_weightonly", (True, False)),
    ("sd_tiny_w4_weightonly", (False, False)),    # full-precision state: planes of the fp32 weights
], ids=["ddim_int8", "sd_tiny_int8", "ddim_weight_only", "sd_tiny_weight_only", "sd_tiny_full_precision"])
def test_reload_lowers_the_new_checkpoint(fake, name, state):
    g = load_case(name)
    ckpt_b = _scaled(g["ckpt"])
    qnn = _fresh(g, g["ckpt"], state)
    d_a = _lower(fake, qnn, g)
    assert qnn._wcache
    import qdiff_b200 as qd
    qd.resume_cali_model(qnn, ckpt_b, None, quant_act=g["qcfg"]["quant_act"])
    qnn.set_quant_state(*state)
    d_reload = _lower(fake, qnn, g)
    d_b = _lower(fake, _fresh(g, ckpt_b, state), g)
    assert d_b != d_a, "the scaled checkpoint must lower to another program"
    assert d_reload == d_b, "after resume_cali_model the model still lowers weights folded from the previous checkpoint"


def test_load_state_dict_drops_folded_weights(fake):
    """QuantModel.load_state_dict (fp32 weights changed in the full-precision state) behaves like a fresh model."""
    g = load_case("sd_tiny_w4_weightonly")
    state = (False, False)
    qnn = _fresh(g, g["ckpt"], state)
    d_a = _lower(fake, qnn, g)
    fresh_b = _fresh(g, _scaled(g["ckpt"]), state)
    qnn.load_state_dict(fresh_b.state_dict())
    d_b = _lower(fake, fresh_b, g)
    assert d_b != d_a
    assert _lower(fake, qnn, g) == d_b


@pytest.mark.parametrize("name", ["sd_tiny_w4a8_sm16", "ddim_w4a8_split"])
def test_state_toggling_matches_fresh_models(fake, name):
    """(True, True) -> (True, False) -> (False, False) -> (True, True) on one model: each lowering equals a fresh model's
    in that state, and coming back to the first state gives the first program again."""
    g = load_case(name)
    seq = [(True, True), (True, False), (False, False), (True, True)]
    qnn = build_qnn(g, CPU)
    got = []
    for state in seq:
        qnn.set_quant_state(*state)
        got.append(_lower(fake, qnn, g))
    for state, d in zip(seq, got):
        assert d == _lower(fake, _fresh(g, g["ckpt"], state), g), state
    assert got[0] == got[3] and len(set(got[:3])) == 3
