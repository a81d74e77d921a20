"""Host-side schedule arithmetic for the fused CFG + DPM-Solver++(2M) device kernel (mos_cfg_dpmpp_step).

Mirrors the scheduler the reference drives at mixofshow/pipelines/pipeline_edlora.py:249,274,290 (diffusers
DPMSolverMultistepScheduler: dpmsolver++, order 2, midpoint, lower_order_final, epsilon prediction, scaled_linear
betas) and DDPMScheduler.add_noise (trainer_edlora.py:218).  Everything here is float64 numpy on the host; the
per-step update itself runs on the GPU.
"""
import json
import os

import numpy as np

# scheduler_config.json settings the fused step hard-codes, with the value it computes.  A config that sets one of them
# to anything else asks for a sampler this class does not implement.
FIXED_CONFIG = {'beta_schedule': 'scaled_linear', 'trained_betas': None, 'prediction_type': 'epsilon', 'solver_order': 2,
                'algorithm_type': 'dpmsolver++', 'solver_type': 'midpoint', 'lower_order_final': True,
                'thresholding': False, 'use_karras_sigmas': False, 'timestep_spacing': 'linspace'}


def alphas_cumprod(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012):
    betas = np.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=np.float32) ** 2
    return np.cumprod((1.0 - betas).astype(np.float32), dtype=np.float32).astype(np.float64)


class DPMSolverPP2M:
    order = 1
    init_noise_sigma = 1.0

    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012):
        ac = alphas_cumprod(num_train_timesteps, beta_start, beta_end)
        self.num_train_timesteps = num_train_timesteps
        self.alpha_t = np.sqrt(ac)
        self.sigma_t = np.sqrt(1.0 - ac)
        self.lambda_t = np.log(self.alpha_t) - np.log(self.sigma_t)
        self.timesteps = None

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, subfolder='scheduler'):
        """diffusers call shape (`DPMSolverMultistepScheduler.from_pretrained(path, subfolder='scheduler')`,
        test_edlora.py:92): takes `num_train_timesteps`, `beta_start` and `beta_end` from `scheduler_config.json` (an SD1.5
        PNDM config included; its PNDM-only keys do not apply here) and rejects every setting in FIXED_CONFIG that differs
        from what this class computes.  Without the file: the SD1.5 defaults."""
        path = os.path.join(pretrained_model_name_or_path, subfolder or '', 'scheduler_config.json')
        if not os.path.isfile(path):
            return cls()
        with open(path) as f:
            cfg = json.load(f)
        for key, value in FIXED_CONFIG.items():
            if key in cfg and cfg[key] != value:
                raise ValueError(f'{path}: {key}={cfg[key]!r} is not supported; the fused DPM-Solver++(2M) step '
                                 f'computes {key}={value!r}')
        return cls(num_train_timesteps=int(cfg.get('num_train_timesteps', 1000)),
                   beta_start=float(cfg.get('beta_start', 0.00085)), beta_end=float(cfg.get('beta_end', 0.012)))

    def set_timesteps(self, num_inference_steps, device=None):
        ts = np.linspace(0, self.num_train_timesteps - 1, num_inference_steps + 1).round()[::-1][:-1].copy()
        ts = ts.astype(np.int64)
        _, uniq = np.unique(ts, return_index=True)
        self.timesteps = ts[np.sort(uniq)]
        return self.timesteps

    def coefficients(self, i):
        """(c_x, c_m0, c_m1, alpha_s, sigma_s):  x0 = (x - sigma_s eps)/alpha_s ; prev = c_x x + c_m0 x0 + c_m1 x0_prev."""
        ts = self.timesteps
        n = len(ts)
        t = int(ts[i])
        prev_t = 0 if i == n - 1 else int(ts[i + 1])
        first_order = i == 0 or (i == n - 1 and n < 15)
        lam_t, lam_s = self.lambda_t[prev_t], self.lambda_t[t]
        a_t, s_t, s_s = self.alpha_t[prev_t], self.sigma_t[prev_t], self.sigma_t[t]
        h = lam_t - lam_s
        c_x = s_t / s_s
        e = a_t * (np.exp(-h) - 1.0)
        if first_order:
            return float(c_x), float(-e), 0.0, float(self.alpha_t[t]), float(s_s)
        h0 = lam_s - self.lambda_t[int(ts[i - 1])]
        r0 = h0 / h
        return float(c_x), float(-e - 0.5 * e / r0), float(0.5 * e / r0), float(self.alpha_t[t]), float(s_s)
