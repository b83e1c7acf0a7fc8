"""Whole N-step tile solves as ONE CUDA graph.

The reference's per-tile loop (training/evaluation/sample_diffusion_decoder.py:105-120; world_pipeline.py:934-949)
runs, per step: precondition_inputs, trigflow_precondition_noise, cat, the U-Net, scheduler.step -- thousands of
launches and host-side scalar math.  Here the step sequence is planned once: the scaled-sample/cond concat is folded
into the first convolution, scheduler.step into the last one, and the per-step scalars (c_in, t, c_skip, c_out, r, k)
sit in a small device table, so a K-step solve of a batch of tiles is a single graph launch of ~80*K kernels.
"""
from __future__ import annotations

import torch

from ..models.plan import UNetEmitter, UNetProgram


def check_plannable(fw, what: str = "model"):
    """The implicit-GEMM convolutions take multiples of 64 channels: name the first layer that is not (e.g. the
    32 / 96-channel layers of the decoder's 32x3 guide) instead of failing inside the planner."""
    for b in fw.enc + fw.dec:
        if b["cout"] % 64:
            raise NotImplementedError(f"{what}: layer {b['name']} has {b['cout']} channels; the implicit-GEMM "
                                      "convolution supports multiples of 64 only")


def fold_score_scaling(row: dict, sigma: float, sigma_data: float, alpha: float) -> dict:
    """Fold the EDM score scaling of sample_diffusion_decoder.py:7-40 (`_scale_score`) into a coefficient row.
    _scale_score is linear in the sample x and the model output F: with t = atan(sigma / sigma_d), c = cos t,
    s = sin t it returns a*x + b*F, a = s(1-c)(1-alpha)/sigma_d, b = c^2 + alpha s^2, so the update's
    x0 = c_skip*x + c_out*(a*x + b*F) is the unscaled update with c_skip += c_out*a, c_out *= b (fp64).
    alpha == 1 returns the row unchanged: c^2 + s^2 is not exactly 1 in floating point."""
    if alpha == 1.0:
        return dict(row)
    import math
    t = math.atan(float(sigma) / float(sigma_data))
    c, s = math.cos(t), math.sin(t)
    a = s * (1.0 - c) * (1.0 - alpha) / float(sigma_data)
    b = c * c + alpha * s * s
    out = dict(row)
    out["c_skip"] = row["c_skip"] + row["c_out"] * a
    out["c_out"] = row["c_out"] * b
    return out


class DiffusionSolve:
    """K-step EDM DPM-Solver++ solve of `n` independent tiles: sample[n, Cs, h, w] (<- noise*sigma0), cond[n, Cc, h, w].

    With a guide model (two-model autoguidance, sample_diffusion_decoder.py:112-117, sample_diffusion_base.py:105-110)
    every step runs the guide's forward first into a solve-owned fp32 buffer, then the main model's forward, whose last
    convolution combines F = F_g + s*(F_m - F_g) before the fused update.  guide=None or guidance_scale == 1 plans
    exactly the unguided program (the reference skips the guide forward then too)."""

    def __init__(self, model, scheduler, n: int, h: int, w: int, num_steps: int, step_range=None, coef_rows=None,
                 guide=None, guidance_scale: float = 1.0, score_scaling: float = 1.0, batch_invariant: bool = False,
                 plan_images: int = 1):
        """coef_rows: explicit per-step tables [dict(c_in, t, c_skip, c_out, r, k)] instead of a scheduler's (the
        TrigFlow consistency step is the same fused program with other numbers: consistency_rows()).
        step_range = (i0, i1): only steps i0 .. i1-1 of the `num_steps` schedule (one PHASE of a multi-phase
        InfiniteDiffusion solve, inference/multiphase.py).  A range that starts in the middle of the schedule starts
        from a blended canvas, so the multistep history is empty there: its first step is first order, exactly like
        a scheduler whose state was reset and positioned at step i0.
        guide / guidance_scale: two-model guidance; score_scaling: the EDM score scaling alpha of the reference's
        decoder sampler, folded into the coefficient rows (fold_score_scaling).
        batch_invariant: each of the n tiles comes out bit-identical to a one-tile solve of it: the launches use their
        one-image item shapes (UNetEmitter), and the host embedding is computed for one tile and shared, so every
        conditional input of run() must then be a single row.  A model that embeds its noise labels on the device
        (the decoder) needs nothing more: the embed launch computes every row on its own.
        plan_images: the image count a batch-invariant solve plans its launches at (UNetEmitter); every solve with the
        same anchor gives a tile the same bits.  A caller that computes each row's embedding on the device itself
        (the latent stage, stages.latent_embedding) writes `emb_all` and calls run(..., embedding_ready=True)."""
        if plan_images != 1 and not batch_invariant:
            raise ValueError("plan_images applies to batch-invariant solves only")
        fw = model.folded()
        dev = fw.device
        self.guided = guide is not None and float(guidance_scale) != 1.0
        self.guide, self.guidance_scale = (guide if self.guided else None), float(guidance_scale)
        if score_scaling != 1.0 and coef_rows is not None:
            raise ValueError("score_scaling applies to scheduler solves, not to explicit coefficient rows")
        if coef_rows is not None:
            co = [dict(r) for r in coef_rows]
            self.schedule_steps, self.step_range = len(co), (0, len(co))
            num_steps = len(co)
        else:
            scheduler.set_timesteps(num_steps)
            order = scheduler.order_schedule()
            i0, i1 = (0, num_steps) if step_range is None else (int(step_range[0]), int(step_range[1]))
            if not (0 <= i0 < i1 <= num_steps):
                raise ValueError(f"step_range {step_range} is not inside the {num_steps}-step schedule")
            self.schedule_steps, self.step_range = num_steps, (i0, i1)
            co = [scheduler.step_coefficients(i, order[i] and not (i == i0 and i0 > 0)) for i in range(i0, i1)]
            if score_scaling != 1.0:
                sd = float(scheduler.config.sigma_data)
                co = [fold_score_scaling(c, float(scheduler.sigmas.double()[i]), sd, float(score_scaling))
                      for c, i in zip(co, range(i0, i1))]
            num_steps = i1 - i0                  # from here on: the number of steps this solve runs
        self.model, self.n, self.h, self.w, self.num_steps = model, n, h, w, num_steps
        self.batch_invariant = batch_invariant
        cs = fw.out_channels
        cc = fw.in_channels - cs
        if self.guided:
            gfw = guide.folded()
            if (gfw.in_channels, gfw.out_channels) != (fw.in_channels, fw.out_channels):
                raise ValueError(f"guide model has {gfw.in_channels} -> {gfw.out_channels} channels; the main model "
                                 f"{fw.in_channels} -> {fw.out_channels}")
            if (len(guide.conditional_layers) > 0 or not gfw.pos_emb) != (len(model.conditional_layers) > 0
                                                                         or not fw.pos_emb):
                raise ValueError("guide and main model must both take host-computed embeddings or neither")
        gcol = [[self.guidance_scale]] * len(co) if self.guided else [[]] * len(co)
        self.coef = torch.tensor([[c["c_skip"], c["c_out"], c["r"], c["k"]] + gc for c, gc in zip(co, gcol)],
                                 dtype=torch.float64).to(torch.float32).to(dev).contiguous()
        self.c_in = torch.tensor([c["c_in"] for c in co], dtype=torch.float64).to(torch.float32).to(dev).contiguous()
        self.labels = torch.tensor([[c["t"]] * n for c in co], dtype=torch.float64).to(torch.float32).to(
            dev).contiguous()
        self.sample = torch.zeros((n, cs, h, w), dtype=torch.float32, device=dev)
        self.cond = torch.zeros((n, max(cc, 1), h, w), dtype=torch.float32, device=dev)
        self.x0_prev = torch.zeros_like(self.sample)
        self.prog = UNetProgram(fw.device)
        # the noise labels of all steps are known up front: ONE embed launch produces every step's modulation vectors
        em = UNetEmitter(fw, n, h, w, cvec_sets=num_steps, batch_invariant=batch_invariant, plan_images=plan_images)
        self.host_emb = len(model.conditional_layers) > 0 or not fw.pos_emb
        if self.guided:
            check_plannable(gfw, "guide model")
            gem = UNetEmitter(gfw, n, h, w, cvec_sets=num_steps,          # its own arena and modulation vectors
                              batch_invariant=batch_invariant, plan_images=plan_images)
            self.guide_out = torch.zeros_like(self.sample)
        if self.host_emb:
            # conditional models (coarse: five float conditions): the 256-wide embeddings of all steps are computed
            # by host torch ops per run() and handed to the embed launch
            self.emb_all = torch.zeros((num_steps * n, fw.emb_channels), dtype=torch.float32, device=dev)
            em.emit_embed(self.prog, emb_in=self.emb_all)
            if self.guided:
                self.guide_emb_all = torch.zeros((num_steps * n, gfw.emb_channels), dtype=torch.float32, device=dev)
                gem.emit_embed(self.prog, emb_in=self.guide_emb_all)
        else:
            em.emit_embed(self.prog, labels=self.labels.reshape(-1))
            if self.guided:
                gem.emit_embed(self.prog, labels=self.labels.reshape(-1))
        for i in range(num_steps):
            srcs = [(self.sample, cs, self.c_in[i:i + 1])]
            if cc > 0:
                srcs.append((self.cond, cc, None))
            sched = dict(coef=self.coef[i], sample=self.sample, x0_prev=self.x0_prev)
            if self.guided:
                gem.emit(self.prog, srcs, model_out=self.guide_out, sched=None, cvec_set=i)
                sched["guide_out"] = self.guide_out
            em.emit(self.prog, srcs, model_out=None, sched=sched, cvec_set=i)
        if self.guided:
            # prog.arena / prog.cvecs stay the main model's (tools read them); the guide's are kept alive in prog.keep
            self.prog.keep.append(gem.arena)
            self.prog.arena, self.prog.cvecs = em.arena, em.cvecs
        self.launches_per_solve = self.prog.n_launch

    @torch.no_grad()
    def run(self, noise: torch.Tensor, cond: torch.Tensor | None, use_graph: bool = True,
            conditional_inputs=None, embedding_ready: bool = False) -> torch.Tensor:
        """noise: [n, Cs, h, w] initial sample (already scaled by sigma_0); returns the denoised sample (a view of the
        solver's state buffer -- copy it before the next run).  embedding_ready: the caller has written every row of
        `emb_all` itself (device-computed embeddings, one per tile and step), so no host embedding is computed and
        conditional_inputs must be None."""
        if embedding_ready:
            if not self.host_emb or self.guided:
                raise ValueError("embedding_ready needs an unguided solve of a model that takes its embedding rows "
                                 "from emb_all")
            if conditional_inputs is not None:
                raise ValueError("embedding_ready: the embedding rows already hold the conditional inputs")
        elif self.host_emb:
            # conditional models: ONE batched evaluation of compute_embeddings for the labels of all steps
            labels = self.labels[:, :1].reshape(-1) if self.batch_invariant else self.labels.reshape(-1)
            if self.batch_invariant and any(c.shape[0] != 1 for c in (conditional_inputs or [])):
                raise ValueError("a batch-invariant solve shares its conditional inputs: pass one row each")
            ci = [c.to(self.labels.device).repeat(self.num_steps, *([1] * (c.dim() - 1)))
                  for c in (conditional_inputs or [])]
            self._set_embedding(self.emb_all, self.model._host_embedding(labels, ci))
            if self.guided:
                self._set_embedding(self.guide_emb_all, self.guide._host_embedding(labels, ci))
        self.sample.copy_(noise)
        if cond is not None:
            self.cond.copy_(cond)
        self.x0_prev.zero_()
        self.prog.run(use_graph)
        return self.sample

    def _set_embedding(self, dst: torch.Tensor, emb: torch.Tensor) -> None:
        """dst [num_steps * n, E] (step-major) <- emb: the same rows, or with batch_invariant one row per step that
        every tile shares (the host GEMMs then see the one-tile shape, whatever n is)."""
        if self.batch_invariant:
            dst.view(self.num_steps, self.n, -1).copy_(emb.view(self.num_steps, 1, -1).expand(-1, self.n, -1))
        else:
            dst.copy_(emb)


def consistency_rows(t: float, sigma_data: float = 0.5, from_unit_noise: bool = False, out_scale: float = 1.0):
    """Coefficient row that makes the fused step program a TrigFlow consistency step
    (world_pipeline.py:1097-1128,1235-1239):   model_in = x_t / sigma_d ;  s' = cos t * x_t + sin t * sigma_d * F
    (pred = -F).  from_unit_noise: the sample buffer holds the unit-variance noise z of a FIRST phase (s = 0, so
    x_t = sin t * sigma_d * z): the re-noising folds into the scalars and no mixing launch is needed.  out_scale
    multiplies the result (1 / sigma_d for a final phase)."""
    import math
    ct, st = math.cos(t), math.sin(t)
    s = st * sigma_data if from_unit_noise else 1.0
    return [dict(c_in=s / sigma_data, t=float(t), c_skip=ct * s * out_scale, c_out=st * sigma_data * out_scale, r=0.0,
                 k=0.0)]
