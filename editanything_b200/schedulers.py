"""Schedulers behind the surface the pipeline uses (`set_timesteps / timesteps / init_noise_sigma /
scale_model_input / step(...).prev_sample / add_noise / order / config`, utils/stable_diffusion_controlnet_inpaint.py:
1430-1431,1012,1547,1634,1651,1538).

`UniPCMultistepScheduler` is what every reference entry point installs (`pipe.scheduler =
UniPCMultistepScheduler.from_config(pipe.scheduler.config)`, editany_lora.py:383,418).  The algorithm lives in
diffusers (pinned 0.17.1 in the reference's environment.yaml:35; NOT vendored and absent from this container), so
this is a restatement of the published UniPC method (Zhao et al. 2023, "UniPC: A Unified Predictor-Corrector
Framework", B(h) = expm1(h) variant "bh2", data-prediction form) with diffusers' defaults: solver_order 2,
predict_x0, lower_order_final, corrector on every step but the first, the last `order` steps falling back to lower
order.  **Parity unpinned** against diffusers itself; pinned here by its invariants (tests/test_schedulers_cpu.py):
order 1 without corrector IS the DDIM eta = 0 update; exactness on x0-linear trajectories; convergence order.

Every update is a linear combination of a few tensors with coefficients that depend on the timestep table only, so
`UniPCMultistepScheduler.coefficient_rows()` exports them for the fused device-side update (DenoiseEngine).
"""
import math
from types import SimpleNamespace

import numpy as np
import torch

from .ops import PREDICTION_TYPES


def _scaled_linear_alphas_cumprod(beta_start, beta_end, n, schedule="scaled_linear"):
    if schedule == "scaled_linear":
        betas = np.linspace(beta_start ** 0.5, beta_end ** 0.5, n, dtype=np.float64) ** 2
    elif schedule == "linear":
        betas = np.linspace(beta_start, beta_end, n, dtype=np.float64)
    else:
        raise NotImplementedError(f"beta_schedule {schedule}")
    return np.cumprod(1.0 - betas, axis=0)


class UniPCMultistepScheduler:
    order = 1
    init_noise_sigma = 1.0

    def __init__(self, num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear",
                 solver_order=2, prediction_type="epsilon", thresholding=False, predict_x0=True, solver_type="bh2",
                 lower_order_final=True, disable_corrector=(), **_ignored):
        if prediction_type not in PREDICTION_TYPES or thresholding or not predict_x0:
            raise NotImplementedError("only epsilon or v prediction in data-prediction (x0) form without thresholding")
        if solver_type not in ("bh1", "bh2"):
            raise NotImplementedError(solver_type)
        self.config = SimpleNamespace(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                                      beta_schedule=beta_schedule, solver_order=solver_order,
                                      prediction_type=prediction_type, thresholding=thresholding, predict_x0=predict_x0,
                                      solver_type=solver_type, lower_order_final=lower_order_final,
                                      disable_corrector=list(disable_corrector))
        self.alphas_cumprod = _scaled_linear_alphas_cumprod(beta_start, beta_end, num_train_timesteps, beta_schedule)
        self.alpha_t = np.sqrt(self.alphas_cumprod)
        self.sigma_t = np.sqrt(1.0 - self.alphas_cumprod)
        self.lambda_t = np.log(self.alpha_t) - np.log(self.sigma_t)
        self.timesteps = None
        self._reset()

    @classmethod
    def from_config(cls, config, **kw):
        """`config`: another scheduler's `.config` (namespace / dict) - the shared keys carry over."""
        src = dict(config) if isinstance(config, dict) else dict(vars(config))
        keep = ("num_train_timesteps", "beta_start", "beta_end", "beta_schedule", "prediction_type")
        args = {k: src[k] for k in keep if k in src}
        args.update(kw)
        return cls(**args)

    def _reset(self):
        k = self.config.solver_order
        self.model_outputs = [None] * k
        self.timestep_list = [None] * k
        self.lower_order_nums = 0
        self.last_sample = None
        self.this_order = 1

    def set_timesteps(self, num_inference_steps, device=None):
        n = self.config.num_train_timesteps
        ts = np.linspace(0, n - 1, num_inference_steps + 1).round()[::-1][:-1].copy().astype(np.int64)
        _, idx = np.unique(ts, return_index=True)        # drop duplicates, keep the descending order
        ts = ts[np.sort(idx)]
        self.timesteps = torch.as_tensor(ts, dtype=torch.long)
        self.num_inference_steps = len(ts)
        self._reset()

    def scale_model_input(self, sample, t):
        return sample

    def add_noise(self, original, noise, timesteps):
        t = int(timesteps.reshape(-1)[0]) if torch.is_tensor(timesteps) else int(timesteps)
        return float(self.alpha_t[t]) * original + float(self.sigma_t[t]) * noise

    # ---- coefficients (pure functions of the timestep table) ---------------------------------------------------
    def _bh_terms(self, t, s0, order, history):
        """Shared by predictor and corrector: h, rks, the R matrix / b vector and the phi terms for the step s0 -> t
        with `history` = the earlier timesteps [s1, s2, ...] (most recent first)."""
        lam_t, lam_s0 = self.lambda_t[t], self.lambda_t[s0]
        h = lam_t - lam_s0
        rks = [(self.lambda_t[si] - lam_s0) / h for si in history[:order - 1]] + [1.0]
        hh = -h
        h_phi_1 = math.expm1(hh)
        h_phi_k = h_phi_1 / hh - 1.0
        B_h = hh if self.config.solver_type == "bh1" else math.expm1(hh)
        R, b, fact = [], [], 1
        for i in range(1, order + 1):
            R.append([rk ** (i - 1) for rk in rks])
            b.append(h_phi_k * fact / B_h)
            fact *= i + 1
            h_phi_k = h_phi_k / hh - 1.0 / fact
        return rks, np.asarray(R, dtype=np.float64), np.asarray(b, dtype=np.float64), h_phi_1, B_h

    def _predictor_coefs(self, t, s0, order, history):
        """x_t = cx * x + c0 * m0 + sum_i ci * m_i   (m0 = newest x0 prediction, m_i = older ones)."""
        rks, R, b, h_phi_1, B_h = self._bh_terms(t, s0, order, history)
        a_t, s_t, s_s0 = self.alpha_t[t], self.sigma_t[t], self.sigma_t[s0]
        cx, c0, cm = s_t / s_s0, -a_t * h_phi_1, [0.0] * (order - 1)
        if order >= 2:
            rhos = np.array([0.5]) if order == 2 else np.linalg.solve(R[:-1, :-1], b[:-1])
            for i in range(order - 1):            # D1_i = (m_i - m0) / rk_i
                w = -a_t * B_h * rhos[i] / rks[i]
                cm[i] += w
                c0 -= w
        return cx, c0, cm

    def _corrector_coefs(self, t, s0, order, history):
        """x_t^c = cx * last_sample + c0 * m0 + sum_i ci * m_i + ct * model_t (model_t = x0 prediction AT t)."""
        rks, R, b, h_phi_1, B_h = self._bh_terms(t, s0, order, history)
        a_t, s_t, s_s0 = self.alpha_t[t], self.sigma_t[t], self.sigma_t[s0]
        rhos = np.array([0.5]) if order == 1 else np.linalg.solve(R, b)
        cx, c0, cm = s_t / s_s0, -a_t * h_phi_1, [0.0] * (order - 1)
        for i in range(order - 1):
            w = -a_t * B_h * rhos[i] / rks[i]
            cm[i] += w
            c0 -= w
        ct = -a_t * B_h * rhos[-1]               # D1_t = model_t - m0
        c0 -= ct
        return cx, c0, cm, ct

    # ---- the stateful step (diffusers surface) -----------------------------------------------------------------
    def step(self, model_output, timestep, sample, **kw):
        if self.timesteps is None:
            raise ValueError("set_timesteps first")
        t = int(timestep)
        hits = (self.timesteps == t).nonzero()
        step_index = len(self.timesteps) - 1 if len(hits) == 0 else int(hits[0])
        k = self.config.solver_order
        use_corrector = (step_index > 0 and (step_index - 1) not in self.config.disable_corrector
                         and self.last_sample is not None)
        if self.config.prediction_type == "v_prediction":                                   # convert_model_output
            x0 = float(self.alpha_t[t]) * sample - float(self.sigma_t[t]) * model_output
        else:
            x0 = (sample - float(self.sigma_t[t]) * model_output) / float(self.alpha_t[t])
        if use_corrector:
            s0 = self.timestep_list[-1]
            hist = [ts for ts in self.timestep_list[-2::-1] if ts is not None]
            cx, c0, cm, ct = self._corrector_coefs(t, s0, self.this_order, hist)
            xc = cx * self.last_sample + c0 * self.model_outputs[-1] + ct * x0
            for i, c in enumerate(cm):
                xc = xc + c * self.model_outputs[-(i + 2)]
            sample = xc.to(sample.dtype)
        prev_t = 0 if step_index == len(self.timesteps) - 1 else int(self.timesteps[step_index + 1])
        for i in range(k - 1):
            self.model_outputs[i] = self.model_outputs[i + 1]
            self.timestep_list[i] = self.timestep_list[i + 1]
        self.model_outputs[-1] = x0
        self.timestep_list[-1] = t
        this_order = min(k, len(self.timesteps) - step_index) if self.config.lower_order_final else k
        self.this_order = min(this_order, self.lower_order_nums + 1)          # warm-up for the multistep
        self.last_sample = sample
        hist = [ts for ts in self.timestep_list[-2::-1] if ts is not None]
        cx, c0, cm = self._predictor_coefs(prev_t, t, self.this_order, hist)
        prev = cx * sample + c0 * x0
        for i, c in enumerate(cm):
            prev = prev + c * self.model_outputs[-(i + 2)]
        if self.lower_order_nums < k:
            self.lower_order_nums += 1
        return SimpleNamespace(prev_sample=prev.to(sample.dtype), pred_original_sample=x0)

    # ---- the same loop as a coefficient table (device-side fused update) ----------------------------------------
    def coefficient_rows(self):
        """One row per step for solver_order <= 2, in terms of the tensors a fused update holds:
            x0  = (x - sigma * eps) / alpha, or alpha * x - sigma * v  (x = latents entering the step)
            xc  = kx * x + kl * last + k1 * m1 + k2 * m2 + k0 * x0     (corrected sample; identity on step 0)
            x'  = px * xc + p0 * x0 + p1 * m1                          (prediction for the next timestep)
            then  m2 <- m1,  m1 <- x0,  last <- xc.
        Returns a list of dicts with keys alpha, sigma, kx, kl, k1, k2, k0, px, p0, p1."""
        if self.config.solver_order > 2:
            raise NotImplementedError("fused update: solver_order <= 2")
        k = self.config.solver_order
        ts = [int(t) for t in self.timesteps]
        rows, t_list, lower = [], [], 0
        this_order = 1
        for i, t in enumerate(ts):
            row = dict(alpha=float(self.alpha_t[t]), sigma=float(self.sigma_t[t]), kx=1.0, kl=0.0, k1=0.0, k2=0.0, k0=0.0)
            if i > 0 and (i - 1) not in self.config.disable_corrector:
                s0 = t_list[-1]
                hist = t_list[-2::-1]
                cx, c0, cm, ct = self._corrector_coefs(t, s0, this_order, hist)
                row.update(kx=0.0, kl=float(cx), k1=float(c0), k2=float(cm[0]) if cm else 0.0, k0=float(ct))
            prev_t = 0 if i == len(ts) - 1 else ts[i + 1]
            t_list = (t_list + [t])[-k:]
            this_order = min(k, len(ts) - i) if self.config.lower_order_final else k
            this_order = min(this_order, lower + 1)
            hist = t_list[-2::-1]
            cx, c0, cm = self._predictor_coefs(prev_t, t, this_order, hist)
            row.update(px=float(cx), p0=float(c0), p1=float(cm[0]) if cm else 0.0)
            if lower < k:
                lower += 1
            rows.append(row)
        return rows
