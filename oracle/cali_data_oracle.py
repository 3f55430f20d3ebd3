"""ORACLE (test infrastructure only): CPU restatement of how the reference's calibration selects its data from a
`--cali_data_path` file: qdiff/utils.py:get_train_samples, the `cali_st > 1` branch (:331-348).  Pinned to the reference
by tests/test_cali_data_cpu.py (fixture tests/golden/cali_data_reader.pt, written by tools/make_cali_data_golden.py
around the reference's own function)."""
import torch


def select_steps(nsteps, cali_st):
    """Indices of the recorded sampling steps the reader uses: every (nsteps // cali_st)-th, starting at step 0."""
    return list(range(0, nsteps, nsteps // cali_st))


def get_train_samples(data, cali_n, cali_st, custom_steps, cond=False):
    """(xs, ts) or, with cond, (xs, ts, conds): the first cali_n samples of each selected step, concatenated in step
    order.  cond doubles xs / ts (the second half pairs with the empty-prompt contexts) and stacks the prompt contexts of
    every selected step, then the empty-prompt ones.  The file must hold at least custom_steps steps."""
    nsteps = len(data["ts"])
    if nsteps < custom_steps:
        raise AssertionError(f"{nsteps} recorded steps < custom_steps {custom_steps}")
    steps = select_steps(nsteps, cali_st)
    xs = [data["xs"][i][:cali_n] for i in steps]
    ts = [data["ts"][i][:cali_n] for i in steps]
    if not cond:
        return torch.cat(xs), torch.cat(ts)
    conds = [data["cs"][i][:cali_n] for i in steps] + [data["ucs"][i][:cali_n] for i in steps]
    return torch.cat(xs + xs), torch.cat(ts + ts), torch.cat(conds)
