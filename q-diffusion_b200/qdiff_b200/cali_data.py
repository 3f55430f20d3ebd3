"""Timestep-aware calibration data (Q-Diffusion section 4.2): the inputs (x_t, t[, c]) of every sampling step of the
full-precision model's own denoising run, in the file format the reference's calibration reads
(qdiff/utils.py:get_train_samples, the `cali_st > 1` branch; `--cali_data_path` of its three scripts):

    {"xs":  [S x fp32 [N, C, H, W]]   entry i: the UNet input of sampling step i (i = 0: x_T at the largest timestep)
     "ts":  [S x [N]]                 the timesteps of that call: int64 (LDM / SD samplers), float32 (generalized_steps)
     "cs":  [S x [N, 77, D]]          conditional runs: each sample's prompt embedding       } one tensor object,
     "ucs": [S x [N, 77, D]]          conditional runs: the empty-prompt embedding           } repeated S times
     "meta": {...}}                   provenance (family, sampler, steps, eta, scale, seed, N, prompts); not read

Every entry of "cs" (and of "ucs") is the same tensor object, so torch.save stores it once.  The reader's `cali_st == 1`
branch (utils.py:328-330) slices the file itself as one tensor; no command of the reference's README uses it, and this
format does not serve it.

Recording: StepRecorder is the `record` callback of samplers.DDIMSampler / PLMSSampler.sample and
samplers.generalized_steps for one batch.  Each step's x and t are copied into device buffers allocated on the batch's
first step, so the loop never waits for the host; CaliData.add gathers the ranks' shards and copies to the host once per
batch.
"""
import os

import torch

from . import dist as qdist


class StepRecorder:
    """record(i, x, t) for one batch of a sampler loop with `steps` steps.  After the loop, .xs is [n, steps, C, H, W]
    fp32 and .ts [n, steps] (the dtype of the loop's t), both on the loop's device."""

    def __init__(self, steps):
        self.steps, self.calls, self.xs, self.ts = int(steps), 0, None, None

    def __call__(self, i, x, t):
        if self.xs is None:
            self.xs = torch.empty((x.shape[0], self.steps) + tuple(x.shape[1:]), dtype=torch.float32, device=x.device)
            self.ts = torch.empty((t.shape[0], self.steps), dtype=t.dtype, device=t.device)
        self.xs[:, i].copy_(x)
        self.ts[:, i].copy_(t)
        self.calls += 1


class CaliData:
    """The calibration set of a run, batch by batch, in sample order.  Every rank calls add() for every batch (it
    gathers); only rank 0 keeps the host copies and writes the file."""

    def __init__(self, rank=0, world=1):
        self.rank, self.world = rank, world
        self.xs, self.ts, self.cs, self.ucs = [], [], [], []

    def add(self, rec, c=None, uc=None):
        """rec: this rank's StepRecorder of the batch.  c / uc: the WHOLE batch's prompt and empty-prompt embeddings
        [B, 77, D] (every rank holds them), or None for unconditional models."""
        if rec.calls != rec.steps:
            raise RuntimeError(f"the sampler recorded {rec.calls} steps, expected {rec.steps}")
        xs, ts = qdist.gather_latents(rec.xs, self.world), qdist.gather_latents(rec.ts, self.world)
        if self.rank != 0:
            return
        self.xs.append(xs.cpu())
        self.ts.append(ts.cpu())
        if c is not None:
            self.cs.append(c.detach().float().cpu())
            self.ucs.append(uc.detach().float().expand(c.shape[0], -1, -1).cpu())

    def state(self, meta):
        steps = self.xs[0].shape[1]
        out = dict(xs=[torch.cat([b[:, i] for b in self.xs]) for i in range(steps)],
                   ts=[torch.cat([b[:, i] for b in self.ts]) for i in range(steps)])
        if self.cs:
            cs, ucs = torch.cat(self.cs), torch.cat(self.ucs)
            out["cs"], out["ucs"] = [cs] * steps, [ucs] * steps
        out["meta"] = dict(meta, N=int(out["xs"][0].shape[0]))
        return out

    def save(self, path, meta):
        """Writes the file on rank 0; returns the path there, None on other ranks."""
        if self.rank != 0:
            return None
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        state = self.state(meta)
        torch.save(state, path)
        print(f"calibration data: {len(state['xs'])} steps x {tuple(state['xs'][0].shape)}"
              f"{' + contexts' if 'cs' in state else ''} -> {path}")
        return path
