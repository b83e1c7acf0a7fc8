"""EDMDPMSolverMultistepScheduler -- drop-in for terrain_diffusion.scheduler.dpmsolver (reference dpmsolver.py:74-762)
for the option set every shipped pipeline uses: algorithm "dpmsolver++", solver "midpoint", order <= 2, karras or
exponential sigmas, prediction "epsilon" / "v_prediction", final_sigmas "zero" / "sigma_min".

Host side (this file): sigma / timestep tables with the reference's fp32 op order (bit-identical tables), step-index
bookkeeping, the order schedule, and the closed-form update coefficients (fp64 -> fp32, SURVEY.md Appendix B).
Device side: ONE vectorised kernel per step (tdx_sched_step) instead of ~25 tiny ATen launches with CPU scalars; the
tile samplers fuse even that into the last convolution (see inference/solve.py).  No CPU fallback for `step`.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import torch

from .. import _lib as L


@dataclass
class SchedulerOutput:
    prev_sample: torch.Tensor


class _AttrDict(dict):
    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e


class EDMDPMSolverMultistepScheduler:
    order = 1

    def __init__(self, sigma_min: float = 0.002, sigma_max: float = 80.0, sigma_data: float = 0.5,
                 scaling_p: float = None, scaling_t: float = 0.05, sigma_schedule: str = "karras",
                 num_train_timesteps: int = 1000, prediction_type: str = "epsilon", rho: float = 7.0,
                 solver_order: int = 2, thresholding: bool = False, dynamic_thresholding_ratio: float = 0.995,
                 sample_max_value: float = 1.0, algorithm_type: str = "dpmsolver++", solver_type: str = "midpoint",
                 lower_order_final: bool = True, euler_at_final: bool = False,
                 final_sigmas_type: Optional[str] = "zero"):
        if algorithm_type == "deis":
            algorithm_type = "dpmsolver++"
        if solver_type in ("logrho", "bh1", "bh2"):
            solver_type = "midpoint"
        if algorithm_type != "dpmsolver++" or solver_type != "midpoint" or solver_order not in (1, 2) or thresholding:
            raise NotImplementedError(
                f"algorithm_type={algorithm_type!r}, solver_type={solver_type!r}, solver_order={solver_order}, "
                f"thresholding={thresholding}: only dpmsolver++ / midpoint / order<=2 / no thresholding (the shipped "
                "configuration) is implemented on the GPU path")
        if prediction_type not in ("epsilon", "v_prediction"):
            raise ValueError(f"Prediction type {prediction_type} is not supported.")
        self._internal_dict = _AttrDict(
            sigma_min=sigma_min, sigma_max=sigma_max, sigma_data=sigma_data, scaling_p=scaling_p, scaling_t=scaling_t,
            sigma_schedule=sigma_schedule, num_train_timesteps=num_train_timesteps, prediction_type=prediction_type,
            rho=rho, solver_order=solver_order, thresholding=thresholding,
            dynamic_thresholding_ratio=dynamic_thresholding_ratio, sample_max_value=sample_max_value,
            algorithm_type=algorithm_type, solver_type=solver_type, lower_order_final=lower_order_final,
            euler_at_final=euler_at_final, final_sigmas_type=final_sigmas_type)
        ramp = torch.linspace(0, 1, num_train_timesteps)
        sigmas = self._compute_sigmas(ramp)
        self.timesteps = self.precondition_noise(sigmas)
        self.sigmas = torch.cat([sigmas, torch.zeros(1)]).to("cpu")
        self.num_inference_steps = None
        self._reset_state()

    # ------------------------------------------------------------------ config / tables (host)
    @property
    def config(self):
        return self._internal_dict

    @property
    def init_noise_sigma(self):
        return (self.config.sigma_max ** 2 + 1) ** 0.5

    @property
    def step_index(self):
        return self._step_index

    @property
    def begin_index(self):
        return self._begin_index

    def set_begin_index(self, begin_index: int = 0):
        self._begin_index = begin_index

    def _reset_state(self):
        self._x0_prev = None
        self.lower_order_nums = 0
        self._step_index = None
        self._begin_index = None

    def _compute_sigmas(self, ramp):
        c = self.config
        if c.sigma_schedule == "karras":
            min_inv_rho = c.sigma_min ** (1 / c.rho)
            max_inv_rho = c.sigma_max ** (1 / c.rho)
            sigmas = (max_inv_rho + ramp * (min_inv_rho - max_inv_rho)) ** c.rho
            if c.scaling_p is not None:
                u = (sigmas - c.sigma_min) / (c.sigma_max - c.sigma_min)
                base = torch.sqrt(torch.maximum(torch.zeros_like(u), 1 - u ** c.scaling_p))
                sigmas = sigmas / (base * (1 - c.scaling_t) + c.scaling_t)
            return sigmas
        if c.sigma_schedule == "exponential":
            return torch.linspace(math.log(c.sigma_min), math.log(c.sigma_max), len(ramp)).exp().flip(0)
        raise ValueError(f"unknown sigma_schedule {c.sigma_schedule!r}")

    def set_timesteps(self, num_inference_steps: int = None, device=None):
        self.num_inference_steps = num_inference_steps
        ramp = torch.linspace(0, 1, num_inference_steps)
        sigmas = self._compute_sigmas(ramp).to(dtype=torch.float32)
        self.timesteps = self.precondition_noise(sigmas)
        if device is not None:
            self.timesteps = self.timesteps.to(device)
        if self.config.final_sigmas_type == "sigma_min":
            last = self.config.sigma_min
        elif self.config.final_sigmas_type == "zero":
            last = 0
        else:
            raise ValueError("`final_sigmas_type` must be one of 'zero', or 'sigma_min', but got "
                             f"{self.config.final_sigmas_type}")
        self.sigmas = torch.cat([sigmas, torch.tensor([last], dtype=torch.float32)]).to("cpu")
        self._reset_state()

    def precondition_inputs(self, sample, sigma):
        return sample * (1 / ((sigma ** 2 + self.config.sigma_data ** 2) ** 0.5))

    def precondition_noise(self, sigma):
        if not isinstance(sigma, torch.Tensor):
            sigma = torch.tensor([sigma])
        return 0.25 * torch.log(sigma)

    def trigflow_precondition_noise(self, sigma):
        return torch.atan(sigma / self.config.sigma_data)

    def precondition_outputs(self, sample, model_output, sigma):
        sd = self.config.sigma_data
        c_skip = sd ** 2 / (sigma ** 2 + sd ** 2)
        c_out = sigma * sd / (sigma ** 2 + sd ** 2) ** 0.5
        if self.config.prediction_type == "v_prediction":
            c_out = -c_out
        return c_skip * sample + c_out * model_output

    def scale_model_input(self, sample, timestep):
        if self._step_index is None:
            self._init_step_index(timestep)
        return self.precondition_inputs(sample, self.sigmas[self._step_index])

    def index_for_timestep(self, timestep, schedule_timesteps=None):
        """Position of `timestep` in the schedule with the reference's tie rule (dpmsolver.py:618-637): a value that
        occurs twice resolves to its SECOND occurrence, an absent value to the last step."""
        table = self.timesteps if schedule_timesteps is None else schedule_timesteps
        hits = torch.nonzero(table == torch.as_tensor(timestep).to(table.device)).flatten().tolist()
        if not hits:
            return len(self.timesteps) - 1
        return hits[min(1, len(hits) - 1)]

    def _init_step_index(self, timestep):
        self._step_index = self.index_for_timestep(timestep) if self._begin_index is None else self._begin_index

    def __len__(self):
        return self.config.num_train_timesteps

    # ------------------------------------------------------------------ closed-form coefficients
    def step_coefficients(self, i: int, second_order: bool) -> dict:
        """x0 = c_skip*x + c_out*F ;  x' = r*x + (1-r)*x0 + k*(x0 - x0_prev).  fp64 from the fp32 sigma table."""
        sd = float(self.config.sigma_data)
        s = self.sigmas.double()
        si, sn = float(s[i]), float(s[i + 1])
        den = si * si + sd * sd
        c_out = si * sd / math.sqrt(den)
        if self.config.prediction_type == "v_prediction":
            c_out = -c_out
        r = sn / si
        k = 0.0
        if second_order:
            h = math.log(si / sn)
            h0 = math.log(float(s[i - 1]) / si)
            k = 0.5 * (1.0 - r) / (h0 / h)
        return dict(c_in=1.0 / math.sqrt(den), t=math.atan(si / sd), c_skip=sd * sd / den, c_out=c_out, r=r, k=k)

    def order_schedule(self) -> list[bool]:
        """second_order flag per step, as `step` would decide it for a fresh run (dpmsolver.py:689-711)."""
        n = len(self.timesteps)
        c = self.config
        out, lower = [], 0
        for i in range(n):
            final = (i == n - 1) and (c.euler_at_final or (c.lower_order_final and n < 15)
                                      or c.final_sigmas_type == "zero")
            out.append(not (c.solver_order == 1 or lower < 1 or final))
            if lower < c.solver_order:
                lower += 1
        return out

    # ------------------------------------------------------------------ device step
    def step(self, model_output, timestep, sample, generator=None, return_dict: bool = True):
        if self.num_inference_steps is None:
            raise ValueError(
                "Number of inference steps is 'None', you need to run 'set_timesteps' after creating the scheduler")
        if model_output.shape != sample.shape:       # the kernel reads sample.numel() elements of both
            raise ValueError(f"model_output shape {list(model_output.shape)} != sample shape {list(sample.shape)}")
        if sample.device.type != "cuda":
            raise L.TdxError("scheduler.step (GPU path) needs CUDA tensors; there is no CPU fallback")
        if self._step_index is None:
            self._init_step_index(timestep)
        i = self._step_index
        n = len(self.timesteps)
        c = self.config
        final = (i == n - 1) and (c.euler_at_final or (c.lower_order_final and n < 15)
                                  or c.final_sigmas_type == "zero")
        second = not (c.solver_order == 1 or self.lower_order_nums < 1 or final)
        co = self.step_coefficients(i, second)
        x = sample.detach().to(torch.float32).contiguous().clone()
        f = model_output.detach().to(torch.float32).contiguous()
        if self._x0_prev is None or self._x0_prev.shape != x.shape or self._x0_prev.device != x.device:
            self._x0_prev = torch.zeros_like(x)
        L.call(L.lib().tdx_sched_step, x.device, x.data_ptr(), f.data_ptr(), self._x0_prev.data_ptr(), x.numel(),
               co["c_skip"], co["c_out"], co["r"], co["k"])
        if self.lower_order_nums < c.solver_order:
            self.lower_order_nums += 1
        self._step_index += 1
        prev = x.to(sample.dtype)
        if not return_dict:
            return (prev,)
        return SchedulerOutput(prev_sample=prev)
