"""One denoising step as a replayed CUDA graph (SURVEY.md section 8(f)1: the RFLOW step loop on the device).

A step of ``RFLOW.sample`` (reference schedulers/scheduling_rflow_open_sora.py:238-250) is ~3500 kernel launches,
each 2-3 us of host work: on 8 GPUs, where a step is ~65 ms of device time, the launch gaps were ~11 % of the step.
The whole step -- CFG concat, STDiT3.forward (our sm_90a kernels, the DSP peer-store switches, the NCCL gather),
guidance combine and Euler update -- is therefore captured ONCE per distinct control flow and replayed:

  * inputs live in static device buffers (latent z, timestep t, dt, the per-frame x_mask); everything else the
    forward reads (caption, fps, height / width) is the same tensor at every step;
  * the only data-dependent control flow of a step is the PAB skip pattern, an integer function of the timestep
    (pab_mgr.py:54-91): the host evaluates it (``STDiT3.pab_plan``), and the plan is the graph's key -- one graph per
    distinct pattern (12 at the OpenSora defaults), all sharing one memory pool since they never run concurrently;
  * DSP epochs advance on the device (csrc/dsp_common.cuh), so a replay needs no host-side counter.

First occurrence of a key runs eagerly (allocates PAB caches / DSP windows, warms cuDNN), the second is captured, later
ones replay.  ``torch.cuda.graphs`` is the capture mechanism only; every kernel inside is launched through the C-ABI.
"""
from typing import Dict, Optional

import torch

from .pab import pab_mgr


class StepGraph:
    def __init__(self, model, guidance_scale: float, enabled: bool = True):
        self.model = model
        self.guidance_scale = float(guidance_scale)
        self.enabled = enabled
        self._seen: Dict[tuple, int] = {}
        self._graphs: Dict[tuple, torch.cuda.CUDAGraph] = {}
        self._pool = None
        self._static: Dict[tuple, dict] = {}  # per graph: a captured graph reads the buffers it was captured with, for ever
        self.launches_per_graph: Dict[tuple, int] = {}
        self.replays = 0
        self.replayed_launches = 0

    # the arithmetic of one step (reference :238-250), shared by the eager and the captured path
    def _compute(self, z, t, dt, fwd_args, plan):
        z_in = torch.cat([z, z], 0)
        tt = torch.cat([t, t], 0)
        out = self.model(z_in, tt, pab_plan=plan, **fwd_args)
        pred = out.chunk(2, dim=1)[0]
        cond, uncond = pred.chunk(2, dim=0)
        v = uncond + self.guidance_scale * (cond - uncond)
        return z + v * dt[:, None, None, None, None]

    def _key(self, z, t, dt, fwd_args, plan):
        ids = tuple((k, v.data_ptr(), tuple(v.shape), v._version) if torch.is_tensor(v) else (k, repr(v))
                    for k, v in sorted(fwd_args.items()) if k != "x_mask")
        # without PAB the timestep never reaches the host and one graph serves every step
        xm = fwd_args.get("x_mask")
        return (tuple(z.shape), z.dtype, t.dtype, dt.dtype, None if xm is None else (tuple(xm.shape), xm.dtype), plan, ids)

    def step(self, z, t, dt, fwd_args, ts_int: Optional[int] = None):
        """z [1,C,T,H,W], t [1], dt [1] device tensors; fwd_args as RFLOW.step passes them (x_mask may change per step);
        ts_int: the integer timestep for the PAB gate (required when PAB is on: the host must not sync inside)."""
        plan = None
        if pab_mgr.enable_pab():
            if ts_int is None:
                ts_int = int(t[0])
            plan = self.model.pab_plan(ts_int)
        if not self.enabled:
            return self._compute(z, t, dt, fwd_args, plan)
        key = self._key(z, t, dt, fwd_args, plan)
        n = self._seen.get(key, 0)
        self._seen[key] = n + 1
        if n == 0:  # first sight: eager (allocations, lazily built windows, library warm-up)
            return self._compute(z, t, dt, fwd_args, plan)
        # static input buffers belong to the KEY (shape / dtype of z are part of it): the first version kept one set and
        # re-allocated it when z's dtype changed (bf16 initial latent, fp32 after the first Euler update), leaving the
        # already captured graph reading freed memory
        st = self._static.get(key)
        xm = fwd_args.get("x_mask")
        if st is None:
            st = self._static[key] = {"z": torch.empty_like(z), "t": torch.empty_like(t), "dt": torch.empty_like(dt),
                                      "x_mask": None if xm is None else torch.empty_like(xm)}
        st["z"].copy_(z)
        st["t"].copy_(t)
        st["dt"].copy_(dt)
        args = dict(fwd_args)
        if xm is not None:
            st["x_mask"].copy_(xm)
            args["x_mask"] = st["x_mask"]
        from .. import kernels

        g = self._graphs.get(key)
        fresh = g is None
        if g is None:

            g = torch.cuda.CUDAGraph()
            if self._pool is None:
                self._pool = torch.cuda.graph_pool_handle()
            torch.cuda.synchronize()
            l0 = kernels.launch_count()
            with torch.cuda.graph(g, pool=self._pool):
                st_out = self._compute(st["z"], st["t"], st["dt"], args, plan)
            self.launches_per_graph[key] = kernels.launch_count() - l0
            self._graphs[key] = g
            self._outs = getattr(self, "_outs", {})
            self._outs[key] = st_out
        g.replay()
        self.replays += 1
        self.replayed_launches += self.launches_per_graph[key]
        if not fresh:  # the capture itself advanced vsb_launch_count once for these kernels
            kernels.GRAPH_REPLAYED_LAUNCHES += self.launches_per_graph[key]
        return self._outs[key].clone()
