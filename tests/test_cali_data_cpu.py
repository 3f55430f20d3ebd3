"""Calibration-data generation without a GPU: the --b200_cali_data_out flag and its refusals on the three scripts, the
reader oracle against the reference's own get_train_samples (tests/golden/cali_data_reader.pt, tools/make_cali_data_golden.py),
the file qdiff_b200.cali_data writes, and the per-batch shard gather on two gloo ranks."""
import io
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import cali_data_oracle as CO
from qdiff_b200 import cali_data, cli

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cali_data_reader.pt")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PARSERS = {"ddim": (lambda: cli.script_parser(cli.ddim_parser()), cli.run_ddim, ["--config", "none.yml"]),
           "ldm": (lambda: cli.script_parser(cli.ldm_parser()), cli.run_ldm, ["--seed", "1"]),
           "txt2img": (lambda: cli.script_parser(cli.txt2img_parser()), cli.run_txt2img, ["--cond"])}
SCRIPTS = {"ddim": ("sample_diffusion_ddim.py", cli.ddim_parser), "ldm": ("sample_diffusion_ldm.py", cli.ldm_parser),
           "txt2img": ("txt2img.py", cli.txt2img_parser)}


def _no_device(monkeypatch):
    def setup(*a, **k):
        raise AssertionError("device work")
    monkeypatch.setattr(cli, "_setup", setup)


# ------------------------------------------------------------------------------------------------ flag and refusals
@pytest.mark.parametrize("which", sorted(PARSERS))
def test_flag_parses_and_passes_the_scope_check(which, monkeypatch):
    parser, run, base = PARSERS[which]
    a = parser().parse_args(base + ["--b200_cali_data_out", "cali.pt"])
    assert a.b200_cali_data_out == "cali.pt" and not a.ptq
    _no_device(monkeypatch)
    with pytest.raises(AssertionError, match="device work"):       # no --ptq needed: the scope check lets it through
        run(a)
    assert parser().parse_args(base).b200_cali_data_out is None


@pytest.mark.parametrize("which", sorted(PARSERS))
def test_refuses_ptq(which, monkeypatch):
    parser, run, base = PARSERS[which]
    _no_device(monkeypatch)
    for extra in (["--ptq"], ["--ptq", "--quant_mode", "qdiff", "--resume", "--cali_ckpt", "c.pth"]):
        with pytest.raises(SystemExit, match="full-precision model.*drop --ptq"):
            run(parser().parse_args(base + ["--b200_cali_data_out", "cali.pt"] + extra))


@pytest.mark.parametrize("which,extra,name", [
    ("ddim", ["--sample_type", "ddpm_noisy"], "--sample_type ddpm_noisy"),
    ("ddim", ["--sample_type", "dpm_solver"], "--sample_type dpm_solver"),
    ("ldm", ["--dpm"], "--dpm"),
    ("ldm", ["-v"], "-v"),
])
def test_refuses_samplers_without_entries(which, extra, name, monkeypatch):
    parser, run, base = PARSERS[which]
    _no_device(monkeypatch)
    with pytest.raises(SystemExit, match=f"{name} records no calibration entries"):
        run(parser().parse_args(base + ["--b200_cali_data_out", "cali.pt"] + extra))


@pytest.mark.parametrize("which", sorted(SCRIPTS))
def test_scripts_take_the_flag_on_top_of_the_sampling_parser(which):
    """Each script parses its sampling parser plus --b200_cali_data_out; the sampling parser itself is unchanged."""
    import subprocess
    import sys
    script, sampling = SCRIPTS[which]
    plain, full = cli.surface(sampling()), cli.surface(cli.script_parser(sampling()))
    assert "b200_cali_data_out" not in plain and sorted(set(full) - set(plain)) == ["b200_cali_data_out"]
    assert all(full[k] == v for k, v in plain.items())
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", script), "--help"], capture_output=True, text=True,
                       timeout=300, cwd=ROOT)
    assert r.returncode == 0 and "--b200_cali_data_out" in r.stdout, r.stderr[-2000:]


def test_without_the_flag_the_refusals_are_unchanged():
    """Namespaces of the sampling parser (no flag at all) and of the script parser without the flag are sampling runs."""
    with pytest.raises(SystemExit, match="pass --ptq"):
        cli._check_scope(cli.script_parser(cli.ldm_parser()).parse_args("--seed 1".split()))
    a = cli.ldm_parser().parse_args("--seed 1".split())
    with pytest.raises(SystemExit, match="pass --ptq"):
        cli._check_scope(a)
    b = cli.txt2img_parser().parse_args("--cond --ptq --quant_mode qdiff --quant_act".split())
    with pytest.raises(SystemExit, match="calibration is not part of the sampling hot path"):
        cli._check_scope(b)


# ------------------------------------------------------------------------------------------------ reader oracle
@pytest.mark.parametrize("case", ["uncond", "cond"])
def test_reader_oracle_matches_reference(case):
    g = torch.load(GOLD, map_location="cpu", weights_only=False)[case]
    for r in g["runs"]:
        out = CO.get_train_samples(g["data"], r["cali_n"], r["cali_st"], r["custom_steps"], cond=case == "cond")
        assert len(out) == len(r["out"]) == (3 if case == "cond" else 2)
        for a, b in zip(out, r["out"]):
            assert a.dtype == b.dtype and torch.equal(a, b), (case, r["cali_n"], r["cali_st"])
    with pytest.raises(AssertionError):                               # the reader's nsteps >= custom_steps
        CO.get_train_samples(g["data"], 1, 2, len(g["data"]["ts"]) + 1)


# ------------------------------------------------------------------------------------------------ the file
def _record_batch(xs, ts):
    """StepRecorder fed the per-step (x, t) of one batch, as a sampler loop feeds it."""
    rec = cali_data.StepRecorder(len(xs))
    for i, (x, t) in enumerate(zip(xs, ts)):
        rec(i, x, t)
    return rec


def test_file_format_and_shared_contexts():
    g = torch.Generator().manual_seed(0)
    S, B, shape = 4, 3, (4, 5, 5)
    data = cali_data.CaliData()
    batches = []
    for _ in range(2):
        xs = [torch.randn(B, *shape, generator=g) for _ in range(S)]
        ts = [torch.full((B,), 900 - 200 * i, dtype=torch.int64) for i in range(S)]
        c, uc = torch.randn(B, 77, 16, generator=g), torch.randn(1, 77, 16, generator=g)
        data.add(_record_batch(xs, ts), c, uc)
        batches.append((xs, ts, c, uc))
    st = data.state(dict(family="sd", sampler="plms", steps=S))
    assert len(st["xs"]) == len(st["ts"]) == len(st["cs"]) == len(st["ucs"]) == S and st["meta"]["N"] == 2 * B
    for i in range(S):
        assert torch.equal(st["xs"][i], torch.cat([b[0][i] for b in batches]))
        assert st["ts"][i].dtype == torch.int64 and torch.equal(st["ts"][i], torch.cat([b[1][i] for b in batches]))
        assert st["cs"][i] is st["cs"][0] and st["ucs"][i] is st["ucs"][0]
    assert torch.equal(st["cs"][0], torch.cat([b[2] for b in batches]))
    assert torch.equal(st["ucs"][0], torch.cat([b[3].expand(B, -1, -1) for b in batches]))
    buf = io.BytesIO()
    torch.save(st, buf)
    payload = 4 * (S * 2 * B * 100 + 2 * 2 * B * 77 * 16)                # xs + one copy each of cs and ucs, fp32
    assert payload < buf.tell() < payload * 1.1 + 20000
    xs, ts, conds = CO.get_train_samples(torch.load(io.BytesIO(buf.getvalue()), weights_only=False), 2 * B, 2, S, cond=True)
    assert xs.shape == (2 * 2 * 2 * B,) + shape and conds.shape == (2 * 2 * 2 * B, 77, 16)


def test_recorder_counts_steps():
    rec = cali_data.StepRecorder(3)
    rec(0, torch.zeros(2, 1, 2, 2), torch.zeros(2))
    with pytest.raises(RuntimeError, match="recorded 1 steps, expected 3"):
        cali_data.CaliData().add(rec)


# ------------------------------------------------------------------------------------------------ two gloo ranks
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _full_batches(S=3, B=4, n_batches=2):
    g = torch.Generator().manual_seed(21)
    return [([torch.randn(B, 2, 3, 3, generator=g) for _ in range(S)], [torch.rand(B, generator=g) * 999 for _ in range(S)])
            for _ in range(n_batches)]


def _worker(rank, world, port, q):
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path[:0] = [root, os.path.join(root, "q-diffusion_b200")]
    from qdiff_b200 import cali_data as CD
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    data = CD.CaliData(rank, world)
    for xs, ts in _full_batches():
        per = xs[0].shape[0] // world
        sl = slice(rank * per, (rank + 1) * per)
        data.add(_record_batch([x[sl] for x in xs], [t[sl] for t in ts]))
    if rank == 0:
        q.put(data.state({}))
    else:
        assert not data.xs                              # only rank 0 keeps host copies
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_gather_keeps_rank_and_step_order():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = q.get(timeout=120)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    batches = _full_batches()
    for i in range(3):
        assert torch.equal(got["xs"][i], torch.cat([b[0][i] for b in batches]))
        assert got["ts"][i].dtype == torch.float32 and torch.equal(got["ts"][i], torch.cat([b[1][i] for b in batches]))
