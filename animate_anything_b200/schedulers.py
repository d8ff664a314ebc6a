"""Schedulers of the sampling loop (models/pipeline.py:148,166,189; train.py:806) with the diffusers 0.24 surface the
reference touches (`set_timesteps`, `timesteps`, `scale_model_input`, `step`, `add_noise`, `config`, `from_config`,
`order`, `init_noise_sigma`, `alphas`) — plus `step_coefficients(timesteps)`, which expresses every step as

    x0 = k0*x + k1*eps ;   x' = k2*x + k3*eps + k4*x0 + k5*x0_prev

so that CFG + the step + the reference's permute/reshape pair run as ONE kernel (`aab_cfg_scheduler_step`).  The
coefficient tables are computed on the host in float64 from the same formulas as diffusers' `step`.
"""
from __future__ import annotations

import inspect
import math
from typing import List, Optional

import numpy as np
import torch

from .modeling import BaseOutput, FrozenConfig


def _betas(num_train_timesteps, beta_start, beta_end, beta_schedule):
    if beta_schedule == "linear":
        return np.linspace(beta_start, beta_end, num_train_timesteps, dtype=np.float64)
    if beta_schedule == "scaled_linear":
        return np.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=np.float64) ** 2
    raise NotImplementedError(beta_schedule)


class SchedulerOutput(BaseOutput):
    pass


class _Base:
    order = 1
    init_noise_sigma = 1.0

    def _capture(self, local):
        sig = inspect.signature(type(self).__init__).parameters
        self.config = FrozenConfig({k: local[k] for k in sig if k != "self"})

    @classmethod
    def from_config(cls, config, **kw):
        sig = inspect.signature(cls.__init__).parameters
        args = {k: v for k, v in dict(config).items() if k in sig}
        args.update({k: v for k, v in kw.items() if k in sig})
        return cls(**args)

    @classmethod
    def from_pretrained(cls, path, subfolder=None, **kw):
        """diffusers SchedulerMixin.from_pretrained (train.py:87 `DDPMScheduler.from_pretrained(path, subfolder="scheduler")`):
        reads `scheduler_config.json`; keys the class does not know (and `_class_name` etc.) are ignored."""
        import json
        import os
        root = os.path.join(path, subfolder) if subfolder else path
        with open(os.path.join(root, "scheduler_config.json")) as f:
            cfg = {k: v for k, v in json.load(f).items() if not k.startswith("_")}
        return cls.from_config(cfg, **kw)

    def save_pretrained(self, path):
        import json
        import os
        os.makedirs(path, exist_ok=True)
        cfg = {k: (list(v) if isinstance(v, tuple) else v) for k, v in self.config.items()}
        cfg["_class_name"] = type(self).__name__
        with open(os.path.join(path, "scheduler_config.json"), "w") as f:
            json.dump(cfg, f, indent=2)

    def _init_tables(self):
        c = self.config
        # float32 tables like diffusers (torch.linspace(..., dtype=float32)) so that indices/values agree
        if c.beta_schedule == "scaled_linear":
            betas = torch.linspace(c.beta_start ** 0.5, c.beta_end ** 0.5, c.num_train_timesteps, dtype=torch.float32) ** 2
        else:
            betas = torch.linspace(c.beta_start, c.beta_end, c.num_train_timesteps, dtype=torch.float32)
        self.betas = betas
        self.alphas = 1.0 - betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)

    def scale_model_input(self, sample, timestep=None):
        return sample

    def add_noise(self, original_samples, noise, timesteps):
        """x_t = sqrt(a_t) x_0 + sqrt(1-a_t) eps  (used once before the loop by utils/common.py:47)."""
        ac = self.alphas_cumprod.to(device=original_samples.device, dtype=original_samples.dtype)
        t = timesteps.to(original_samples.device).long()
        sa = (ac[t] ** 0.5).flatten()
        sb = ((1 - ac[t]) ** 0.5).flatten()
        while sa.dim() < original_samples.dim():
            sa, sb = sa.unsqueeze(-1), sb.unsqueeze(-1)
        return sa * original_samples + sb * noise

    def step(self, model_output, timestep, sample, **kw):
        raise NotImplementedError("this pipeline fuses CFG + scheduler step into one kernel "
                                  "(LatentToVideoPipeline / ops.cfg_scheduler_step with step_coefficients()); "
                                  "a stand-alone torch step() is deliberately not provided")


class DDIMScheduler(_Base):
    def __init__(self, num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear",
                 clip_sample=True, set_alpha_to_one=True, steps_offset=0, prediction_type="epsilon",
                 thresholding=False, clip_sample_range=1.0, timestep_spacing="leading"):
        self._capture(locals())
        self._init_tables()
        self.final_alpha_cumprod = torch.tensor(1.0) if set_alpha_to_one else self.alphas_cumprod[0]
        self.num_inference_steps = None
        self.timesteps = torch.from_numpy(np.arange(0, num_train_timesteps)[::-1].copy().astype(np.int64))

    def set_timesteps(self, num_inference_steps, device=None):
        c = self.config
        self.num_inference_steps = num_inference_steps
        if c.timestep_spacing == "linspace":
            ts = np.linspace(0, c.num_train_timesteps - 1, num_inference_steps).round()[::-1].copy().astype(np.int64)
        elif c.timestep_spacing == "leading":
            ratio = c.num_train_timesteps // num_inference_steps
            ts = (np.arange(0, num_inference_steps) * ratio).round()[::-1].copy().astype(np.int64) + c.steps_offset
        elif c.timestep_spacing == "trailing":
            ratio = c.num_train_timesteps / num_inference_steps
            ts = np.round(np.arange(c.num_train_timesteps, 0, -ratio)).astype(np.int64) - 1
        else:
            raise ValueError(c.timestep_spacing)
        self.timesteps = torch.from_numpy(ts).to(device)

    def step_coefficients(self, timesteps, eta: float = 0.0, _continue=False):
        c = self.config
        if eta != 0.0:
            raise NotImplementedError("stochastic DDIM (eta > 0) is not fused; the reference calls with eta=0.0")
        if c.clip_sample or c.thresholding:
            raise NotImplementedError("clip_sample / thresholding are not fused (ModelScope config: clip_sample=False)")
        ac = self.alphas_cumprod.double().numpy()
        rows = []
        for t in timesteps:
            t = int(t)
            prev_t = t - c.num_train_timesteps // self.num_inference_steps
            a_t = ac[t]
            a_p = ac[prev_t] if prev_t >= 0 else float(self.final_alpha_cumprod)
            sa, sb = math.sqrt(a_t), math.sqrt(1 - a_t)
            if c.prediction_type == "epsilon":
                rows.append([1 / sa, -sb / sa, 0.0, math.sqrt(1 - a_p), math.sqrt(a_p), 0.0])
            elif c.prediction_type == "v_prediction":
                rows.append([sa, -sb, math.sqrt(1 - a_p) * sb, math.sqrt(1 - a_p) * sa, math.sqrt(a_p), 0.0])
            else:
                raise NotImplementedError(c.prediction_type)
        return np.asarray(rows, dtype=np.float32), False     # (table, needs x0 history)


class DDPMScheduler(DDIMScheduler):
    """Only the surface train.py:86 / utils/common.py:32-48 need (tables, timesteps, add_noise)."""

    def __init__(self, num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear",
                 variance_type="fixed_small", clip_sample=True, prediction_type="epsilon", timestep_spacing="leading",
                 steps_offset=0):
        self._capture(locals())
        self._init_tables()
        self.final_alpha_cumprod = torch.tensor(1.0)
        self.num_inference_steps = None
        self.timesteps = torch.from_numpy(np.arange(0, num_train_timesteps)[::-1].copy().astype(np.int64))

    def step_coefficients(self, *a, **k):
        raise NotImplementedError("ancestral DDPM sampling is not on the reference's eval path")


class DPMSolverMultistepScheduler(_Base):
    """dpmsolver++ / midpoint / order 2 / lower_order_final — what `DPMSolverMultistepScheduler.from_config(
    pipeline.scheduler.config)` at train.py:806 yields."""

    def __init__(self, num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear",
                 solver_order=2, prediction_type="epsilon", thresholding=False, algorithm_type="dpmsolver++",
                 solver_type="midpoint", lower_order_final=True, use_karras_sigmas=False,
                 lambda_min_clipped=-float("inf"), timestep_spacing="linspace", steps_offset=0):
        self._capture(locals())
        if algorithm_type != "dpmsolver++" or solver_type != "midpoint" or solver_order not in (1, 2) or \
                use_karras_sigmas or thresholding:
            raise NotImplementedError("only dpmsolver++ / midpoint / order<=2 (the reference's configuration)")
        self._init_tables()
        self.num_inference_steps = None
        self.timesteps = torch.from_numpy(np.linspace(0, num_train_timesteps - 1, num_train_timesteps)[::-1].copy()
                                          .astype(np.int64))
        self.sigmas = None

    def set_timesteps(self, num_inference_steps, device=None):
        c = self.config
        ac = self.alphas_cumprod
        lambda_t = torch.log(torch.sqrt(ac)) - torch.log(torch.sqrt(1 - ac))
        clipped_idx = torch.searchsorted(torch.flip(lambda_t, [0]), c.lambda_min_clipped)
        last = int((c.num_train_timesteps - clipped_idx).item())
        if c.timestep_spacing == "linspace":
            ts = np.linspace(0, last - 1, num_inference_steps + 1).round()[::-1][:-1].copy().astype(np.int64)
        elif c.timestep_spacing == "leading":
            ratio = last // (num_inference_steps + 1)
            ts = (np.arange(0, num_inference_steps + 1) * ratio).round()[::-1][:-1].copy().astype(np.int64) + c.steps_offset
        elif c.timestep_spacing == "trailing":
            ratio = c.num_train_timesteps / num_inference_steps
            ts = np.arange(last, 0, -ratio).round().copy().astype(np.int64) - 1
        else:
            raise ValueError(c.timestep_spacing)
        sig = (((1 - ac) / ac) ** 0.5).numpy()
        sig = np.interp(ts, np.arange(0, len(sig)), sig)
        sig_last = float(((1 - ac[0]) / ac[0]) ** 0.5)
        self.sigmas = np.concatenate([sig, [sig_last]]).astype(np.float32).astype(np.float64)
        self.timesteps = torch.from_numpy(ts).to(device=device, dtype=torch.int64)
        self.num_inference_steps = len(ts)

    def step_coefficients(self, timesteps, eta: float = 0.0, _continue=False):
        c = self.config
        all_ts = [int(v) for v in self.timesteps.tolist()]
        n_all = len(all_ts)
        rows = []
        lower_order_nums = 0
        step_index = None
        for t in timesteps:
            t = int(t)
            if step_index is None:        # diffusers _init_step_index
                cand = [i for i, v in enumerate(all_ts) if v == t]
                step_index = (n_all - 1) if not cand else (cand[1] if len(cand) > 1 else cand[0])
            i = step_index

            def a_s(sigma):
                a = 1.0 / math.sqrt(sigma * sigma + 1.0)
                return a, sigma * a
            alpha_s0, sigma_s0 = a_s(self.sigmas[i])
            alpha_t, sigma_t = a_s(self.sigmas[i + 1])
            lam_t = math.log(alpha_t) - math.log(sigma_t)
            lam_s0 = math.log(alpha_s0) - math.log(sigma_s0)
            h = lam_t - lam_s0
            if c.prediction_type == "epsilon":
                k0, k1 = 1.0 / alpha_s0, -sigma_s0 / alpha_s0
            elif c.prediction_type == "v_prediction":
                k0, k1 = alpha_s0, -sigma_s0
            else:
                raise NotImplementedError(c.prediction_type)
            big_a = alpha_t * (math.exp(-h) - 1.0)
            lower_final = (i == n_all - 1) and c.lower_order_final and n_all < 15
            if c.solver_order == 1 or lower_order_nums < 1 or lower_final:
                rows.append([k0, k1, sigma_t / sigma_s0, 0.0, -big_a, 0.0])
            else:
                alpha_s1, sigma_s1 = a_s(self.sigmas[i - 1])
                lam_s1 = math.log(alpha_s1) - math.log(sigma_s1)
                r0 = (lam_s0 - lam_s1) / h
                rows.append([k0, k1, sigma_t / sigma_s0, 0.0, -big_a - 0.5 * big_a / r0, 0.5 * big_a / r0])
            if lower_order_nums < c.solver_order:
                lower_order_nums += 1
            step_index += 1
        return np.asarray(rows, dtype=np.float32), True


class EulerDiscreteScheduler(_Base):
    """Host side of diffusers' EulerDiscreteScheduler as Stable Video Diffusion configures it (v-prediction, Karras sigmas,
    continuous timesteps 0.25 * log(sigma), "leading" spacing; called at models/pipeline.py:412,418,439).  The arithmetic of
    `scale_model_input` / `step` runs in `aab_svd_in_assemble` / `aab_svd_cfg_euler_step`; this class owns the sigma and
    timestep tables (float32, same construction order as diffusers so that the values agree bit for bit with the oracle)."""

    def __init__(self, num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear",
                 prediction_type="epsilon", interpolation_type="linear", use_karras_sigmas=False, sigma_min=None,
                 sigma_max=None, timestep_spacing="linspace", timestep_type="discrete", steps_offset=0):
        self._capture(locals())
        self._init_tables()
        import numpy as np
        sig = np.array(((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5)
        sigmas = torch.from_numpy(sig[::-1].copy()).to(dtype=torch.float32)
        self.sigmas = torch.cat([sigmas, torch.zeros(1)])
        self.timesteps = (torch.Tensor([0.25 * s.log() for s in sigmas]) if self._continuous_v() else
                          torch.from_numpy(np.linspace(0, num_train_timesteps - 1, num_train_timesteps, dtype=float)[::-1].copy()
                                           ).to(torch.float32))
        self.num_inference_steps = None

    def _continuous_v(self):
        return self.config.timestep_type == "continuous" and self.config.prediction_type == "v_prediction"

    @property
    def init_noise_sigma(self):
        m = self.sigmas.max()
        if self.config.timestep_spacing in ("linspace", "trailing"):
            return m
        return (m ** 2 + 1) ** 0.5

    def set_timesteps(self, num_inference_steps, device=None):
        import numpy as np
        c = self.config
        n = c.num_train_timesteps
        self.num_inference_steps = num_inference_steps
        if c.timestep_spacing == "linspace":
            ts = np.linspace(0, n - 1, num_inference_steps, dtype=np.float32)[::-1].copy()
        elif c.timestep_spacing == "leading":
            ts = (np.arange(0, num_inference_steps) * (n // num_inference_steps)).round()[::-1].copy().astype(np.float32)
            ts += c.steps_offset
        else:
            ts = (np.arange(n, 0, -n / num_inference_steps)).round().copy().astype(np.float32) - 1
        sig = np.array(((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5)
        log_sig = np.log(sig)
        sig = np.interp(ts, np.arange(0, len(sig)), sig)
        if c.use_karras_sigmas:
            smin = c.sigma_min if c.sigma_min is not None else sig[-1].item()
            smax = c.sigma_max if c.sigma_max is not None else sig[0].item()
            ramp = np.linspace(0, 1, num_inference_steps)
            sig = (smax ** (1 / 7.0) + ramp * (smin ** (1 / 7.0) - smax ** (1 / 7.0))) ** 7.0
            ts = np.array([self._sigma_to_t(s_, log_sig) for s_ in sig])
        sigmas = torch.from_numpy(sig).to(dtype=torch.float32)
        if self._continuous_v():
            self.timesteps = torch.Tensor([0.25 * s_.log() for s_ in sigmas]).to(device=device)
        else:
            self.timesteps = torch.from_numpy(np.asarray(ts, dtype=np.float32)).to(device=device)
        self.sigmas = torch.cat([sigmas, torch.zeros(1)])

    @staticmethod
    def _sigma_to_t(sigma, log_sigmas):
        import numpy as np
        log_sigma = np.log(np.maximum(sigma, 1e-10))
        dists = log_sigma - log_sigmas[:, np.newaxis]
        low_idx = np.cumsum((dists >= 0), axis=0).argmax(axis=0).clip(max=log_sigmas.shape[0] - 2)
        high_idx = low_idx + 1
        low, high = log_sigmas[low_idx], log_sigmas[high_idx]
        w = np.clip((low - log_sigma) / (low - high), 0, 1)
        return ((1 - w) * low_idx + w * high_idx).reshape(sigma.shape)

    def step_coefficients(self, *a, **k):
        raise NotImplementedError("Euler steps are fused in aab_svd_cfg_euler_step (pipeline_svd.py)")
