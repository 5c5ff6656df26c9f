"""DDPM / DDIM / F-PNDM reverse-diffusion loops with the reference's signatures.

Drop-in for ``ddpm_sampler`` / ``ddim_sampler`` / ``FPNDM_sampler`` of the reference
``models/__init__.py:207-340, 103-203, 39-99`` (+ ``models/pndm.py``): same keyword arguments
(unknown ones are swallowed, exactly like the reference's ``**kwargs``), same return shape
``[1 or T, B, C*F, S, S]`` on the input's device.

The loop keeps the state ``x`` in a static NCHW device buffer; each step launches the lowered network
program and one fused update kernel (x0-prediction, clamp, posterior mean, + sigma * z) -- nothing is
synchronised with the host unless ``log`` / ``verbose`` ask for the reference's diagnostics.
Schedule coefficients are computed with the same fp32 torch expressions as the reference so they are
bit-identical.
"""
from __future__ import annotations

import logging
from typing import List, Optional

import numpy as np
import torch

from . import lib
from .model import UNetMore_DDPM


def _unwrap(scorenet) -> UNetMore_DDPM:
    net = scorenet.module if hasattr(scorenet, "module") else scorenet
    if not isinstance(net, UNetMore_DDPM):
        raise TypeError("mcvd_b200 samplers drive mcvd_b200.UNetMore_DDPM modules "
                        f"(got {type(net).__name__}); use the reference samplers for reference modules")
    return net


def _schedule(net, subsample_steps):
    """models/__init__.py:211-240 on CPU fp32 tensors (values identical to the reference's)."""
    alphas, alphas_prev, betas = net.alphas.detach().cpu(), net.alphas_prev.detach().cpu(), net.betas.detach().cpu()
    steps = np.arange(len(betas))
    if subsample_steps is not None and subsample_steps < len(alphas):
        skip = len(alphas) // subsample_steps
        steps = torch.tensor(list(range(0, len(alphas), skip)))
        alphas = alphas.index_select(0, steps)
        alphas_prev = torch.cat([alphas[1:], torch.tensor([1.0])])
        betas = 1.0 - torch.div(alphas, alphas_prev)
    return steps, alphas, alphas_prev, betas


class _Loop:
    """Shared plumbing: program lookup, input staging, per-step launch."""

    def __init__(self, x_mod, scorenet, cond):
        self.net = _unwrap(scorenet)
        self.eng = self.net.engine()
        # the engine refuses to exist off-GPU (no CPU fallback); a CPU x_mod is staged to its device and the
        # result is returned on x_mod's device, as the reference samplers do
        self.dev = self.eng.device
        self.out_dev = x_mod.device              # results go back to the caller's device (reference contract)
        self.B = x_mod.shape[0]
        self.shape = x_mod.shape
        self.launches = 0
        if self.eng.spec.cond_ch > 0 and cond is None:
            raise RuntimeError("mcvd_b200: cond is required by this network")
        self._ctx = self.eng._devctx()
        self._ctx.__enter__()
        try:                                     # anything below may raise (build failure, OOM): do not leak the
            self.P = self.eng.program(self.B)    # current-device context
            self.eng.set_inputs(self.P, x=x_mod.to(self.dev).float(),
                                cond=None if cond is None else cond.to(self.dev).float())
            self.eng.run_cond(self.P)
            self.launches += self.P.cond_launches
            self.u = self.P.update_arr[0]
        except BaseException:
            self._ctx.__exit__(None, None, None)
            raise

    def close(self):
        self._ctx.__exit__(None, None, None)

    def result(self, t):
        return t.to(self.out_dev)

    def eps(self, t):
        """eps = net(x_state, t, cond) into P.eps_nhwc (x_state = P.x_in)."""
        self.eng.set_inputs(self.P, t=t)
        self.eng.run_step_graphed(self.P)
        self.launches += self.P.step_launches

    def update(self, k0, k1, ca, cb, cc, sigma, clip, noise=None, philox=None, step=0):
        u = self.u
        u.f0, u.f1, u.f2, u.f3, u.f4, u.f5 = float(k0), float(k1), float(ca), float(cb), float(cc), float(sigma)
        fl = lib.F_CLIP if clip else 0
        if sigma != 0.0:
            if philox is not None:
                seed, clip0 = philox
                fl |= lib.F_PHILOX
                u.i0, u.i1, u.i2, u.i3 = int(seed & 0x7FFFFFFF), int((seed >> 31) & 0x7FFFFFFF), int(clip0), int(step)
            else:
                self.P.noise.copy_(noise.reshape(self.P.noise.shape))
        u.flags = fl
        self.eng._run(self.P.update_arr, 1)
        self.launches += 1

    def state(self):
        return self.P.x_in.reshape(self.shape).clone()

    def eps_nchw(self):
        self.eng._run(self.P.out_arr, 1)
        self.launches += 1
        return self.P.out.reshape(self.shape)


def _log_line(tag, i, L, grad, x, c_alpha, verbose, log):
    """Diagnostics of models/__init__.py:295-308 (forces host syncs, as in the reference)."""
    g = -1 / (1 - c_alpha).sqrt().item() * grad
    grad_norm = torch.norm(g.reshape(g.shape[0], -1), dim=-1).mean()
    image_norm = torch.norm(x.reshape(x.shape[0], -1), dim=-1).mean()
    grad_mean_norm = torch.norm(g.mean(dim=0).reshape(-1)) ** 2 * (1 - c_alpha).item()
    msg = "{}: {}/{}, grad_norm: {}, image_norm: {}, grad_mean_norm: {}".format(
        tag, i + 1, L, grad_norm.item(), image_norm.item(), grad_mean_norm.item())
    if verbose:
        print(msg)
    if log:
        logging.info(msg)


@torch.no_grad()
def ddpm_sampler(x_mod, scorenet, cond=None, just_beta=False, final_only=False, denoise=True, subsample_steps=None,
                 same_noise=False, noise_val=None, frac_steps=None, verbose=False, log=False, clip_before=True,
                 t_min=-1, gamma=False, noise_list: Optional[List[torch.Tensor]] = None, philox_seed=None,
                 clip_offset=0, warm_noise: Optional[torch.Tensor] = None, **kwargs):
    """Reference ``ddpm_sampler`` (models/__init__.py:207-340).

    Extensions (keyword-only in practice): ``noise_list`` = per-step injected noise (L-1 tensors) for
    parity tests; ``philox_seed`` / ``clip_offset`` = draw the noise in-kernel from a counter-based
    stream keyed by the GLOBAL clip index, so a clip gets the same noise on any GPU.  With neither, the
    noise is ``torch.randn_like`` as in the reference (:324).
    """
    if gamma:
        raise NotImplementedError("gamma=True is not accelerated (reference models/__init__.py:214,319-322)")
    t_min = -1 if t_min is None else t_min
    lp = _Loop(x_mod, scorenet, cond)
    try:
        steps, alphas, alphas_prev, betas = _schedule(lp.net, subsample_steps)
        if frac_steps is not None:                                             # :249-256
            steps = steps[int((1 - frac_steps) * len(steps)):]
            alphas, alphas_prev, betas = alphas[steps], alphas_prev[steps], betas[steps]
        if same_noise and noise_val is None:                                    # :258-259
            noise_val = x_mod.detach().clone()
        L = len(steps)
        images = []
        x_transf = False
        for i, step in enumerate(steps):
            if step < t_min * len(alphas):                                      # :269-270 (init_prev_t warm start)
                continue
            if not x_transf and t_min > 0:                                      # :272-279: noise x to this level
                z0 = warm_noise if warm_noise is not None else torch.randn(lp.P.noise.shape, device=lp.dev)
                lp.update(0.0, 0.0, 0.0, alphas[i].sqrt().item(), 0.0, (1 - alphas[i]).sqrt().item(), False, noise=z0)
            x_transf = True
            c_beta, c_alpha, c_alpha_prev = betas[i], alphas[i], alphas_prev[i]
            lp.eps(float(step))                                                 # :283-284
            k0 = 1 / c_alpha.sqrt()                                             # :287
            k1 = (1 - c_alpha).sqrt()
            ca = c_alpha_prev.sqrt() * c_beta / (1 - c_alpha)                   # :290
            cb = (1 - c_beta).sqrt() * (1 - c_alpha_prev) / (1 - c_alpha)
            last = i + 1 == L
            sigma, noise = 0.0, None
            if not last:                                                        # :311-328
                sigma = (c_beta.sqrt() if just_beta else ((1 - c_alpha_prev) / (1 - c_alpha) * c_beta).sqrt()).item()
                if same_noise:
                    noise = noise_val
                elif noise_list is not None:
                    noise = noise_list[i]
                elif philox_seed is None:
                    noise = torch.randn(lp.P.noise.shape, device=lp.dev, dtype=torch.float32)
            want_log = (verbose or log) and (i == 0 or (i + 1) % max(L // 10, 1) == 0)
            if want_log or not final_only:
                # the reference reports / stores x BEFORE the noise is added (:292-308)
                lp.update(k0.item(), k1.item(), ca.item(), cb.item(), 0.0, 0.0, clip_before)
                if not final_only:
                    images.append(lp.state().to("cpu"))
                if want_log:
                    _log_line("DDPM", i, L, lp.eps_nchw(), lp.state(), c_alpha, verbose, log)
                if sigma != 0.0:  # x += sigma * z  == update with x0-coefficient 0 and x-coefficient 1
                    lp.update(0.0, 0.0, 0.0, 1.0, 0.0, sigma, False, noise=noise,
                              philox=None if philox_seed is None or noise is not None else (philox_seed, clip_offset),
                              step=i)
            else:
                lp.update(k0.item(), k1.item(), ca.item(), cb.item(), 0.0, sigma, clip_before, noise=noise,
                          philox=None if philox_seed is None or noise is not None else (philox_seed, clip_offset),
                          step=i)
        if denoise:                                                             # :331-335
            lp.eps(float(L - 1))
            lp.update(0.0, 0.0, 0.0, 1.0, -(1 - alphas[-1]).sqrt().item(), 0.0, False)
            if not final_only:
                images.append(lp.state().to("cpu"))
        ddpm_sampler.last_launches = lp.launches
        if final_only:
            return lp.result(lp.state().unsqueeze(0))
        return torch.stack(images)
    finally:
        lp.close()


@torch.no_grad()
def ddim_sampler(x_mod, scorenet, cond=None, final_only=False, denoise=True, subsample_steps=None, verbose=False,
                 log=True, clip_before=True, t_min=-1, gamma=False, warm_noise: Optional[torch.Tensor] = None, **kwargs):
    """Reference ``ddim_sampler`` (models/__init__.py:103-203): x = sqrt(a_prev) x0 + sqrt(1 - a_prev) eps."""
    if gamma:
        raise NotImplementedError("gamma=True is not accelerated")
    t_min = -1 if t_min is None else t_min
    lp = _Loop(x_mod, scorenet, cond)
    try:
        steps, alphas, alphas_prev, betas = _schedule(lp.net, subsample_steps)
        L = len(steps)
        images = []
        x_transf = False
        for i, step in enumerate(steps):
            if step < t_min * len(alphas):                                           # :143-144
                continue
            if not x_transf and t_min > 0:                                           # :146-153
                z0 = warm_noise if warm_noise is not None else torch.randn(lp.P.noise.shape, device=lp.dev)
                lp.update(0.0, 0.0, 0.0, alphas[i].sqrt().item(), 0.0, (1 - alphas[i]).sqrt().item(), False, noise=z0)
            x_transf = True
            c_alpha, c_alpha_prev = alphas[i], alphas_prev[i]
            lp.eps(float(step))
            lp.update((1 / c_alpha.sqrt()).item(), (1 - c_alpha).sqrt().item(), c_alpha_prev.sqrt().item(), 0.0,
                      (1 - c_alpha_prev).sqrt().item(), 0.0, clip_before)          # :163-166
            if not final_only:
                images.append(lp.state().to("cpu"))
            if (verbose or log) and (i == 0 or (i + 1) % max(L // 10, 1) == 0):
                _log_line("DDIM", i, L, lp.eps_nchw(), lp.state(), c_alpha, verbose, log)
        if denoise:                                                                 # :194-196
            lp.eps(float(L - 1))
            lp.update(0.0, 0.0, 0.0, 1.0, -(1 - alphas[-1]).sqrt().item(), 0.0, False)
            if not final_only:
                images.append(lp.state().to("cpu"))
        if final_only:
            return lp.result(lp.state().unsqueeze(0))
        return torch.stack(images)
    finally:
        lp.close()


@torch.no_grad()
def FPNDM_sampler(x_mod, scorenet, cond=None, final_only=False, denoise=True, subsample_steps=None, verbose=False,
                  log=True, clip_before=True, t_min=-1, gamma=False, **kwargs):
    """Reference ``FPNDM_sampler`` + ``pndm.gen_order_4`` (models/__init__.py:39-99, models/pndm.py:3-52).

    Replicated as written: alphas looked up through the flipped copy with the +1 offset, steps_next =
    [-1] + steps[:-1], fractional mid-timesteps fed to the network, no final denoise call.  Every
    network call (L + 9 of them) runs in the CUDA library; the eps history (``ets``), its 4-term linear
    combination and the per-step ``transfer`` are a handful of tiny elementwise torch ops on the GPU
    (they could be fused into the update kernel).
    """
    lp = _Loop(x_mod, scorenet, cond)
    try:
        net = lp.net
        alphas = net.alphas.detach().cpu()
        alphas_old = alphas.flip(0)                                                  # :58
        skip = len(alphas) // subsample_steps
        steps = list(range(0, len(alphas), skip))
        steps_next = [-1] + steps[:-1]                                               # :63
        P = lp.P

        def eps_at(x, t):
            lp.eng.set_inputs(P, x=x)
            lp.eps(float(t))
            return lp.eps_nchw().clone()

        def transfer(x, t, t_next, et):
            """pndm.py:19-34.  x_next = x + (a' - a) * (cx * x - ce * et), then optional clamp."""
            at = alphas_old[int(t) + 1]
            an = alphas_old[int(t_next) + 1]
            cx = 1 / (at.sqrt() * (at.sqrt() + an.sqrt()))
            ce = 1 / (at.sqrt() * (((1 - an) * at).sqrt() + ((1 - at) * an).sqrt()))
            x_next = x + (an - at) * (cx * x - ce * et)
            return x_next.clip_(-1, 1) if clip_before else x_next

        x = x_mod.to(lp.dev).float()             # eps tensors live on the engine's device; keep x there too
        ets: List[torch.Tensor] = []
        images = []
        for i in range(len(steps)):
            t, t_next = steps[i], steps_next[i]
            t_mid = (t + t_next) / 2                                                 # pndm.py:42 (fractional)
            if len(ets) > 2:                                                         # pndm.py:44-47
                ets.append(eps_at(x, t))
                noise = (1 / 24) * (55 * ets[-1] - 59 * ets[-2] + 37 * ets[-3] - 9 * ets[-4])
            else:                                                                    # runge_kutta, pndm.py:3-17
                e1 = eps_at(x, t)
                ets.append(e1)
                # the alpha lookup truncates the fractional mid-timestep (.long(), pndm.py:20-21)
                tm_idx = int(torch.tensor(t_mid).long().item())
                x2 = transfer(x, t, tm_idx, e1)
                e2 = eps_at(x2, t_mid)
                x3 = transfer(x, t, tm_idx, e2)
                e3 = eps_at(x3, t_mid)
                x4 = transfer(x, t, t_next, e3)
                e4 = eps_at(x4, t_next)
                noise = (1 / 6) * (e1 + 2 * e2 + 2 * e3 + e4)
            x = transfer(x, t, t_next, noise)
            if not final_only:
                images.append(x.to("cpu"))
        if final_only:
            return lp.result(x.reshape(lp.shape).unsqueeze(0))
        return torch.stack(images)
    finally:
        lp.close()


def get_sampler(config):
    """Same dispatch as reference ``NCSNRunner.get_sampler`` (runners/ncsn_runner.py:2702-2714)."""
    from functools import partial
    version = getattr(config.model, "version", "DDPM").upper()
    if version == "DDPM":
        return partial(ddpm_sampler, config=config)
    if version == "DDIM":
        return partial(ddim_sampler, config=config)
    if version == "FPNDM":
        return partial(FPNDM_sampler, config=config)
    raise NotImplementedError(f"sampler for version {version!r} is not part of the accelerated path")
