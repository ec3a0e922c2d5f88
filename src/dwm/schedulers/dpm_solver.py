"""DPM-Solver++ multistep scheduler — the `inference_config["scheduler"]` of the reference's
image example (`diffusers.DPMSolverMultistepScheduler`,
examples/ctsd_21_6views_image_generation.json; instantiated at
src/dwm/pipelines/ctsd.py:981-985, stepped with one scalar timestep per iteration at
:1573-1575).  Restates diffusers==0.31.0 for algorithm_type "dpmsolver++", solver_type
"midpoint", solver_order <= 2, no Karras sigmas / thresholding (diffusers' defaults on top of
the SD-2.1 `scheduler_config.json`).

All per-step coefficients depend only on the sigma table, so `set_timesteps` evaluates them
once (fp64 on the host) and keeps them on the device; a step is then one launch of the fused
CFG + DPM-Solver++ kernel (`dwm_b200_cfg_dpmpp_step`) with no host-device traffic:

    x0   = c_x[i] * sample + c_m[i] * model_output          (epsilon / sample / v_prediction)
    prev = k_s[i] * sample + k_0[i] * x0_i + k_1[i] * x0_{i-1}

The multistep state the kernel reads is on the device: the x0 history (one buffer, updated in
place) and, for a captured CUDA graph, the coefficient row and order of the step (`load_row`).
The host keeps only the counters that pick the row, so a caller that replays a graph loads the
row before each replay and calls `advance` after it.
"""
import json
import math
import os
from dataclasses import dataclass

import numpy as np
import torch

from opendwm_b200 import ops as _ops


class _Config(dict):
    __getattr__ = dict.get


@dataclass
class SchedulerOutput:
    prev_sample: torch.Tensor


class DPMSolverMultistepScheduler:
    order = 1

    def __init__(self, num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02,
                 beta_schedule="linear", trained_betas=None, solver_order=2,
                 prediction_type="epsilon", thresholding=False, algorithm_type="dpmsolver++",
                 solver_type="midpoint", lower_order_final=True, euler_at_final=False,
                 use_karras_sigmas=False, use_lu_lambdas=False, final_sigmas_type="zero",
                 lambda_min_clipped=-float("inf"), variance_type=None,
                 timestep_spacing="linspace", steps_offset=0, **unused):
        if algorithm_type != "dpmsolver++" or solver_type != "midpoint" or solver_order > 2 \
                or thresholding or use_karras_sigmas or use_lu_lambdas \
                or trained_betas is not None or lambda_min_clipped != -float("inf"):
            raise NotImplementedError(
                "only DPM-Solver++ (midpoint, order <= 2, plain sigmas) is provided")
        self.config = _Config(
            num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
            beta_schedule=beta_schedule, solver_order=solver_order,
            prediction_type=prediction_type, algorithm_type=algorithm_type,
            solver_type=solver_type, lower_order_final=lower_order_final,
            euler_at_final=euler_at_final, final_sigmas_type=final_sigmas_type,
            timestep_spacing=timestep_spacing, steps_offset=steps_offset)
        if beta_schedule == "scaled_linear":
            betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps,
                                   dtype=torch.float32) ** 2
        elif beta_schedule == "linear":
            betas = torch.linspace(beta_start, beta_end, num_train_timesteps,
                                   dtype=torch.float32)
        else:
            raise NotImplementedError(beta_schedule)
        self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
        self.init_noise_sigma = 1.0
        self.num_inference_steps = None
        self.timesteps = torch.arange(num_train_timesteps - 1, -1, -1)
        self._begin_index = 0
        self._x0 = self._row = None       # device x0 history and static coefficient row

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, subfolder=None, **kwargs):
        path = pretrained_model_name_or_path
        if subfolder:
            path = os.path.join(path, subfolder)
        with open(os.path.join(path, "scheduler_config.json")) as f:
            cfg = {k: v for k, v in json.load(f).items() if not k.startswith("_")}
        # a DDIM / PNDM style config (SD-2.1 ships one) only contributes the keys this class has
        keep = ("num_train_timesteps", "beta_start", "beta_end", "beta_schedule",
                "trained_betas", "prediction_type", "steps_offset", "timestep_spacing",
                "solver_order", "thresholding", "algorithm_type", "solver_type",
                "lower_order_final", "euler_at_final", "use_karras_sigmas",
                "use_lu_lambdas", "final_sigmas_type", "lambda_min_clipped")
        cfg = {k: v for k, v in cfg.items() if k in keep}
        if cfg.get("timestep_spacing") is None:
            cfg.pop("timestep_spacing", None)
        cfg.update(kwargs)
        return cls(**cfg)

    def scale_model_input(self, sample, timestep=None):
        return sample

    def set_begin_index(self, begin_index: int = 0):
        self._begin_index = begin_index
        self._reset(begin_index)

    def _reset(self, step_index):
        """Starts a fresh multistep history at `step_index`: the next step is first order."""
        self._step_index = step_index
        self.lower_order_nums = 0
        for buf in (self._x0, self._row):
            if buf is not None:
                buf.zero_()

    def set_timesteps(self, num_inference_steps: int, device=None):
        c = self.config
        last = c.num_train_timesteps
        n = num_inference_steps
        if c.timestep_spacing == "linspace":
            ts = np.linspace(0, last - 1, n + 1).round()[::-1][:-1].copy().astype(np.int64)
        elif c.timestep_spacing == "leading":
            ratio = last // (n + 1)
            ts = (np.arange(0, n + 1) * ratio).round()[::-1][:-1].copy().astype(np.int64)
            ts += c.steps_offset
        elif c.timestep_spacing == "trailing":
            ratio = c.num_train_timesteps / n
            ts = np.arange(last, 0, -ratio).round().copy().astype(np.int64) - 1
        else:
            raise ValueError(c.timestep_spacing)
        sig = (((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5).numpy()
        sig = np.interp(ts, np.arange(0, len(sig)), sig)
        last_sigma = 0.0 if c.final_sigmas_type == "zero" else \
            float(((1 - self.alphas_cumprod[0]) / self.alphas_cumprod[0]) ** 0.5)
        sigmas = np.concatenate([sig, [last_sigma]]).astype(np.float32)
        self.sigmas = torch.from_numpy(sigmas)
        self.timesteps = torch.from_numpy(ts).to(device=device, dtype=torch.int64)
        self.num_inference_steps = n
        self._begin_index = 0
        self._coef = self._coefficients(sigmas.astype(np.float64)).to(device)
        self._reset(0)

    def _coefficients(self, s):
        """[n, 2, 6] fp32: for step i and (first-order, second-order) variant the row
        (c_x, c_m, k_s, k_0, k_1, order) of the two linear combinations in the module
        docstring; the kernel adds the k_1 term exactly when order is 2."""
        n = len(s) - 1
        out = np.zeros((n, 2, 6))
        out[:, 0, 5], out[:, 1, 5] = 1.0, 2.0
        alpha = 1.0 / np.sqrt(s * s + 1.0)
        sig = s * alpha

        def lam(j):
            return math.inf if sig[j] == 0 else math.log(alpha[j]) - math.log(sig[j])
        pt = self.config.prediction_type
        for i in range(n):
            if pt == "epsilon":
                cx, cm = 1.0 / alpha[i], -sig[i] / alpha[i]
            elif pt == "sample":
                cx, cm = 0.0, 1.0
            elif pt == "v_prediction":
                cx, cm = alpha[i], -sig[i]
            else:
                raise ValueError(pt)
            h = lam(i + 1) - lam(i)
            e1 = math.expm1(-h) if math.isfinite(h) else -1.0      # exp(-h) - 1
            ks, k = sig[i + 1] / sig[i], -alpha[i + 1] * e1
            out[i, 0, :5] = (cx, cm, ks, k, 0.0)
            if i > 0:
                r0 = (lam(i) - lam(i - 1)) / h if math.isfinite(h) else 0.0
                out[i, 1, :5] = (cx, cm, ks, k * (1.0 + 0.5 / r0), -0.5 * k / r0) if r0 != 0.0 \
                    else out[i, 0, :5]
        return torch.from_numpy(out.astype(np.float32))

    def step(self, model_output, timestep=None, sample=None, generator=None,
             variance_noise=None, return_dict: bool = True):
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run "
                             "'set_timesteps' after creating the scheduler")
        if not model_output.is_cuda:
            raise RuntimeError("scheduler kernels run on CUDA only (no CPU fallback)")
        prev = torch.empty(sample.shape, device=model_output.device, dtype=torch.float32)
        prev.copy_(sample)
        self.cfg_step_(model_output.to(torch.float32).contiguous(), prev, cfg=1)
        prev = prev.to(model_output.dtype)
        if not return_dict:
            return (prev,)
        return SchedulerOutput(prev_sample=prev)

    def cfg_step_(self, pred, latents, guidance_scale=1.0, cfg=2):
        """One step on fp32 `latents` in place from fp32 `pred` [cfg * latents.numel()]
        (unconditional half first when cfg is 2): the CFG combine
        u + guidance_scale * (c - u) and the DPM-Solver++ update in one launch.  Under CUDA-graph
        capture the launch reads the static row buffer, which the replaying caller fills with
        `load_row` before each replay (and calls `advance` after it)."""
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run "
                             "'set_timesteps' after creating the scheduler")
        x0, row = self.device_state(latents)
        if not torch.cuda.is_current_stream_capturing():
            i, variant = self._row_index()
            row = self._coef[i, variant]
        _ops.cfg_dpmpp_step(pred, latents, x0, row, cfg=cfg, guidance_scale=guidance_scale)
        self.advance()
        return latents

    # -- device-state protocol: what a caller replaying the step from a CUDA graph needs ------
    def device_state(self, sample):
        """(x0 history, coefficient row) device buffers for steps on `sample`; allocated on
        first use and kept (a captured graph holds their addresses) until the sample's size or
        device changes, which is only allowed at the start of a schedule."""
        dev = sample.device
        if self._coef.device != dev:
            self._coef = self._coef.to(dev)
        if self._row is None or self._row.device != dev:
            self._row = torch.zeros(6, device=dev)
        if self._x0 is None or self._x0.device != dev or self._x0.numel() != sample.numel():
            if self.lower_order_nums > 0:
                raise ValueError("the sample changed size or device within a schedule; call "
                                 "set_timesteps or set_begin_index first")
            self._x0 = torch.zeros(sample.numel(), device=dev)
        return self._x0, self._row

    def _row_index(self):
        """Host bookkeeping of the next step: (step index, 0 first / 1 second order)."""
        i, c = self._step_index, self.config
        n = len(self.timesteps)
        if not 0 <= i < n:
            raise IndexError("step {} is outside the {}-step schedule".format(i, n))
        lower_final = i == n - 1 and (c.euler_at_final or (c.lower_order_final and n < 15) or
                                      c.final_sigmas_type == "zero")
        first = c.solver_order == 1 or self.lower_order_nums < 1 or lower_final
        return i, 0 if first else 1

    def load_row(self):
        """Copies the next step's coefficient row and order into the static row buffer."""
        i, variant = self._row_index()
        self._row.copy_(self._coef[i, variant])

    def advance(self):
        """Advances the host counters past one step."""
        if self.lower_order_nums < self.config.solver_order:
            self.lower_order_nums += 1
        self._step_index += 1

    def snapshot(self):
        """The multistep state (counters, x0 history, row) for `restore`."""
        return (self._step_index, self.lower_order_nums,
                None if self._x0 is None else self._x0.clone(),
                None if self._row is None else self._row.clone())

    def restore(self, state):
        """Puts back a `snapshot`, in place in the buffers a captured graph reads."""
        self._step_index, self.lower_order_nums, x0, row = state
        for buf, old in ((self._x0, x0), (self._row, row)):
            if buf is not None:
                buf.copy_(old) if old is not None else buf.zero_()
