"""The stage in front of the edit: DDIM inversion of the encoded frames and the on-disk hand-off the drivers read
(reference preprocess.py:198-230 `ddim_inversion`, :232-261 `ddim_sample`, :227-229 / :313-314 the files).

The VAE stage around it is here too (`encode_imgs`, `decode_latents`, reference preprocess.py:163-182 and
run_tokenflow_pnp.py:145-163, on `vae.AutoencoderKL`), and the edit's starting noise (`ddim_eps`, run_tokenflow_pnp.py:
186-193), so that one process goes from uint8 frames to edited uint8 frames without the disk:

    encode_imgs -> LatentInverter.ddim_inversion -> saved_latents() -> ddim_eps -> scheduler.add_noise ->
    TokenFlowEditor.sample_loop -> decode_latents

With a ControlNet (controlnet.py) and the Canny conditioning of the frames (`canny_cond`), every UNet call of both
directions is the reference's `controlnet_pred` (preprocess.py:129-149): the ControlNet on the batch's frames of the
conditioning, then the UNet with its residuals.  The CLIP text encoder and the depth variant stay out of scope.  The
latents directory is still written in the reference's format, so it can be read back by `TokenFlowEditor` / the
reference drivers (`tokenflow_utils.load_source_latents_t`).  Frames are independent in this stage, so with several ranks each rank
inverts its own contiguous share and the saved tensors are all-gathered.

Two paths compute the same steps:
  * CPU / fp32 UNet: the eager loop below, step by step as the reference writes it;
  * CUDA fp16 UNet: one CUDA graph of a step over the rank's share (the UNet calls in batches of `batch_size`, then the
    DDIM update `tf_ddim` in place, `tf_ddim_v` for a v-prediction scheduler), replayed for every step of both
    directions.  The step's timestep and its four DDIM coefficients are read from device buffers the host refreshes per
    replay; saved timesteps are device-to-device copies into one resident buffer, all-gathered once at the end.
"""
from __future__ import annotations

import os
from typing import Dict, Iterable, List, Optional, Tuple

import torch

from .ops import all_gather, frame_share, gather_frames


def inversion_coef_tables(scheduler) -> Tuple[torch.Tensor, torch.Tensor]:
    """fp32 [steps, 4] coefficient rows (s1, inv_s2, s3, s4) of `tf_ddim` for every step of the inversion (ascending
    timesteps) and of the reconstruction (descending), from `scheduler.timesteps` of the grid that is set.

    The values are the ones the reference's expressions produce (preprocess.py:211-224, :245-259): its alphas are 0-dim
    fp32 tensors, so `1 - a` and `a ** 0.5` are fp32 operations, and ATen divides the fp16 latents by the 0-dim
    `mu` as a multiply by the fp32 reciprocal 1 / mu.  `final_alpha_cumprod` stands in for the missing neighbour at
    both ends of the grid.
    inversion step i (t = ts_up[i], prev = ts_up[i - 1]):     sigma_prev, 1 / mu_prev, mu, sigma
    reconstruction step i (t = ts_dn[i], prev = ts_dn[i + 1]): sigma, 1 / mu, mu_prev, sigma_prev

    For a v-prediction scheduler the rows are those of `tf_ddim_v` (diffusers' DDIMInverseScheduler / DDIMScheduler
    v-branch, which multiplies by every coefficient and divides by none), from the same 0-dim fp32 alphas:
    inversion (mu_prev, sigma_prev, mu, sigma), reconstruction (mu, sigma, mu_prev, sigma_prev)."""
    a = scheduler.alphas_cumprod.cpu()
    final = scheduler.final_alpha_cumprod.cpu()
    ts_dn = [int(t) for t in scheduler.timesteps.tolist()]
    ts_up = ts_dn[::-1]
    v = scheduler.prediction_type == "v_prediction"
    # 0-dim CPU tensor arithmetic, one step at a time, exactly as the reference evaluates it (the CPU's fp32 sqrt is
    # ATen's, which need not be the correctly rounded one)
    mu_sigma = lambda alpha: (alpha ** 0.5, (1 - alpha) ** 0.5)
    inv, rec = [], []
    for i, t in enumerate(ts_up):
        mu, sigma = mu_sigma(a[t])
        mu_p, sigma_p = mu_sigma(a[ts_up[i - 1]] if i > 0 else final)
        inv.append(torch.stack([mu_p, sigma_p, mu, sigma] if v else [sigma_p, 1 / mu_p, mu, sigma]))
    for i, t in enumerate(ts_dn):
        mu, sigma = mu_sigma(a[t])
        mu_p, sigma_p = mu_sigma(a[ts_dn[i + 1]] if i < len(ts_dn) - 1 else final)
        rec.append(torch.stack([mu, sigma, mu_p, sigma_p] if v else [sigma, 1 / mu, mu_p, sigma_p]))
    return torch.stack(inv), torch.stack(rec)


def saved_timesteps(ts_up: List[int], timesteps_to_save: Optional[Iterable[int]]) -> List[int]:
    """The timesteps of an inversion over `ts_up` whose latents are saved (reference preprocess.py:227-229): those in
    `timesteps_to_save` (default: all), and the last one."""
    keep = set(int(t) for t in timesteps_to_save) if timesteps_to_save is not None else set(ts_up)
    return [t for i, t in enumerate(ts_up) if t in keep or i == len(ts_up) - 1]


class LatentInverter:
    def __init__(self, unet, scheduler, n_timesteps: int, world_size: int = 1, rank: int = 0, group=None,
                 controlnet=None, controlnet_cond: Optional[torch.Tensor] = None):
        """`scheduler.set_timesteps(n_timesteps)` defines the inversion grid (reference default: 500 steps, of which
        the 50 sampling timesteps are saved).  `controlnet` and `controlnet_cond` ([N, 3, H, W], the Canny
        conditioning of all N frames, `canny_cond`) run every UNet call as the reference's `controlnet_pred`; each
        rank reads the conditioning of its own frames."""
        if (controlnet is None) != (controlnet_cond is None):
            raise ValueError("LatentInverter needs both controlnet and controlnet_cond, or neither")
        self.unet, self.scheduler = unet, scheduler
        self.controlnet, self.controlnet_cond = controlnet, controlnet_cond
        self.device = next(unet.parameters()).device
        self.scheduler.set_timesteps(n_timesteps, device=self.device)
        self.world_size, self.rank, self.group = world_size, rank, group
        self.comm = None                      # ops.Communicator (C-ABI NCCL all-gather), see attach_communicator
        self._saved: Dict[int, torch.Tensor] = {}
        self._graphs = {}                     # (share shape, batch size, cond shape) -> captured step
        self._graph_pool = None
        self._tables = None
        self._use_graph = True                # test seam: False runs the same device path eagerly

    def attach_communicator(self, comm):
        """Route the final all-gather of the graphed path through the C ABI (tf_allgather) instead of
        torch.distributed."""
        self.comm = comm

    def saved_latents(self) -> Dict[int, torch.Tensor]:
        """{t: [N, 4, h, w]} of the last `ddim_inversion` (either path, with `save_latents`) — the tensors it writes as
        `noisy_latents_<t>.pt`, kept in memory so that `TokenFlowEditor(..., source_latents=
        inv.saved_latents().__getitem__)` needs no disk round trip."""
        return self._saved

    # -- the two DDIM directions -------------------------------------------------------------------------------
    def _alphas(self, t: int, t_prev: Optional[int]):
        a_t = float(self.scheduler.alphas_cumprod[t])
        a_prev = float(self.scheduler.alphas_cumprod[t_prev]) if t_prev is not None else float(self.scheduler.final_alpha_cumprod)
        return a_t ** 0.5, (1 - a_t) ** 0.5, a_prev ** 0.5, (1 - a_prev) ** 0.5          # mu, sigma, mu_prev, sigma_prev

    def _eps(self, x, t: int, cond, frame0: int = 0):
        """The UNet's noise prediction for the frames [frame0, frame0 + len(x)) (reference preprocess.py:222-223)."""
        from .controlnet import controlnet_residuals
        t_dev = torch.tensor(t, device=x.device)
        ctx = cond.repeat(x.shape[0], 1, 1)
        ccond = None
        if self.controlnet is not None:
            ccond = self.controlnet_cond[frame0:frame0 + x.shape[0]].to(x.device)
        res = controlnet_residuals(self.controlnet, x, t_dev, ctx, ccond)
        out = self.unet(x, t_dev, encoder_hidden_states=ctx, **res)
        return out["sample"] if isinstance(out, dict) else out.sample

    def _local(self, n: int):
        return frame_share(n, self.world_size, self.rank)

    def _gathered(self, x_local, n: int):
        return gather_frames(x_local, n, self.world_size, self.group, self.comm)

    @torch.no_grad()
    def ddim_inversion(self, cond: torch.Tensor, latent_frames: torch.Tensor, save_path: Optional[str], batch_size: int,
                       save_latents: bool = True, timesteps_to_save: Optional[Iterable[int]] = None) -> torch.Tensor:
        """Reference preprocess.py:198-230.  latent_frames [N,4,h,w] (clean, VAE-encoded) → the latents at the noisiest
        timestep; `noisy_latents_<t>.pt` is written for every t in `timesteps_to_save` (default: all) and for the
        last one."""
        if self._graphed_path():
            return self._device_inversion(cond, latent_frames, save_path, batch_size, save_latents, timesteps_to_save)
        ts = [int(t) for t in reversed(self.scheduler.timesteps.tolist())]                 # ascending noise level
        keep = set(int(t) for t in timesteps_to_save) if timesteps_to_save is not None else set(ts)
        n = latent_frames.shape[0]
        lo, hi = self._local(n)
        x = latent_frames[lo:hi].clone()
        if save_latents and save_path is not None:
            os.makedirs(os.path.join(save_path, "latents"), exist_ok=True)
        self._saved = {}
        for i, t in enumerate(ts):
            mu, sigma, mu_prev, sigma_prev = self._alphas(t, ts[i - 1] if i > 0 else None)
            for b in range(0, x.shape[0], batch_size):
                xb = x[b:b + batch_size]
                x[b:b + batch_size] = self._update(xb, self._eps(xb, t, cond, lo + b), mu_prev, sigma_prev, mu, sigma)
            if save_latents and (t in keep or i == len(ts) - 1):
                full = self._saved[t] = self._gathered(x, n).clone()
                if save_path is not None and self.rank == 0:
                    torch.save(full, os.path.join(save_path, "latents", f"noisy_latents_{t}.pt"))
        return self._gathered(x, n)

    @torch.no_grad()
    def ddim_sample(self, x: torch.Tensor, cond: torch.Tensor, batch_size: int) -> torch.Tensor:
        """Reference preprocess.py:232-261: deterministic DDIM reconstruction from the inverted latents (the
        `inverted.mp4` check of the reference, in latent space)."""
        if self._graphed_path():
            return self._device_sample(x, cond, batch_size)
        ts = [int(t) for t in self.scheduler.timesteps.tolist()]
        n = x.shape[0]
        lo, hi = self._local(n)
        x = x[lo:hi].clone()
        for i, t in enumerate(ts):
            mu, sigma, mu_prev, sigma_prev = self._alphas(t, ts[i + 1] if i < len(ts) - 1 else None)
            for b in range(0, x.shape[0], batch_size):
                xb = x[b:b + batch_size]
                x[b:b + batch_size] = self._update(xb, self._eps(xb, t, cond, lo + b), mu, sigma, mu_prev, sigma_prev)
        return self._gathered(x, n)

    def _update(self, x, m, mu_from, sigma_from, mu_to, sigma_to):
        """One DDIM step of the eager loop from the level of x (mu_from, sigma_from) to the next (mu_to, sigma_to), for
        the model output m: the reference's eps update (preprocess.py:224-225 / :259-260), or for a v-prediction
        scheduler diffusers' DDIMInverseScheduler / DDIMScheduler v-branch (the reference has none)."""
        if self.scheduler.prediction_type == "v_prediction":
            pred_x0 = mu_from * x - sigma_from * m
            pred_eps = mu_from * m + sigma_from * x
            return mu_to * pred_x0 + sigma_to * pred_eps
        pred_x0 = (x - sigma_from * m) / mu_from
        return mu_to * pred_x0 + sigma_to * m

    # -- CUDA fp16: graph-replayed steps ------------------------------------------------------------------------
    def _graphed_path(self) -> bool:
        p = next(self.unet.parameters())
        return p.is_cuda and p.dtype == torch.float16

    def _device_tables(self):
        """(inversion coefficients, reconstruction coefficients, ascending timesteps, descending timesteps) on the
        device, for the grid that is set."""
        ts_dn = [int(t) for t in self.scheduler.timesteps.tolist()]
        if self._tables is None or self._tables[0] != ts_dn:
            inv, rec = inversion_coef_tables(self.scheduler)
            dev = lambda v: v.to(self.device)
            self._tables = (ts_dn, dev(inv), dev(rec), dev(torch.tensor(ts_dn[::-1])), dev(torch.tensor(ts_dn)))
        return self._tables[1:]

    def _step_runner(self, share: int, shape, batch_size: int, cond: torch.Tensor):
        """Static buffers and the step over a share of `share` frames: the UNet over the share in batches of
        `batch_size` (each call preceded by the ControlNet on the batch's conditioning when there is one), then
        `tf_ddim` in place.  Captured once per share shape and replayed; `_use_graph = False` runs the same function
        eagerly."""
        from . import tokenflow_utils as tfu
        from .controlnet import controlnet_residuals
        ops = tfu._ops()                      # the library is required: raises without it or without an H100
        update = ops.ddim_v if self.scheduler.prediction_type == "v_prediction" else ops.ddim
        bs = max(1, min(batch_size, share))
        key = (share, tuple(shape), bs, tuple(cond.shape[1:]), self._use_graph, self.controlnet is not None)
        entry = self._graphs.get(key)
        if entry is not None:
            entry["cond"].copy_(cond.expand(bs, -1, -1))
            return entry
        dev = self.device
        st = {"x": torch.zeros((share,) + tuple(shape), dtype=torch.float16, device=dev),
              "t": torch.zeros((), dtype=torch.int64, device=dev),
              "coef": torch.zeros(4, dtype=torch.float32, device=dev),
              "cond": cond.to(dev, torch.float16).repeat(bs, 1, 1)}
        if self.controlnet is not None:
            # the share's conditioning, refreshed per call by `_run_steps`, in the ControlNet's memory format
            cl = next(self.controlnet.parameters()).is_contiguous(memory_format=torch.channels_last)
            st["ccond"] = torch.zeros((share,) + tuple(self.controlnet_cond.shape[1:]), dtype=torch.float16,
                                      device=dev).contiguous(memory_format=torch.channels_last if cl else
                                                             torch.contiguous_format)

        def step():
            x = st["x"]
            outs = []
            for b in range(0, share, bs):
                xb = x[b:b + bs]
                ctx = st["cond"][:xb.shape[0]]
                res = controlnet_residuals(self.controlnet, xb, st["t"], ctx, st["ccond"][b:b + bs]) \
                    if self.controlnet is not None else {}
                out = self.unet(xb, st["t"], encoder_hidden_states=ctx, **res)
                outs.append(out["sample"] if isinstance(out, dict) else out.sample)
            eps = outs[0] if len(outs) == 1 else torch.cat(outs)
            update(eps, x, st["coef"], out=x)

        entry = {"st": st, "cond": st["cond"], "step": step, "graph": None}
        if self._use_graph and share > 0:
            # warm-up on a side stream (cuDNN autotuning, lazy initialisation, allocator growth), then one capture
            # into the inverter's private pool.  Both run on the zeroed buffers, before the real latents arrive.
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(2):
                    step()
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, pool=self._graph_pool, capture_error_mode="thread_local"):
                step()
            if self._graph_pool is None:
                self._graph_pool = graph.pool()
            entry["graph"] = graph
        self._graphs[key] = entry
        return entry

    def _run_steps(self, x_share: torch.Tensor, cond, batch_size: int, coef: torch.Tensor, ts: torch.Tensor,
                   save_slots: Optional[Dict[int, int]] = None, saved: Optional[torch.Tensor] = None,
                   frame0: int = 0):
        """All steps of one direction over this rank's share: per step, refresh the timestep and the coefficient row,
        replay, and copy the latents of a saved step into its slot of `saved`.  Returns the share's final latents.
        `frame0` is the share's first frame: the ControlNet conditioning is read from there."""
        share = x_share.shape[0]
        if share == 0:
            return x_share
        entry = self._step_runner(share, x_share.shape[1:], batch_size, cond)
        st = entry["st"]
        st["x"].copy_(x_share)
        if "ccond" in st:
            st["ccond"].copy_(self.controlnet_cond[frame0:frame0 + share])
        for i in range(coef.shape[0]):
            st["t"].copy_(ts[i])
            st["coef"].copy_(coef[i])
            if entry["graph"] is not None:
                entry["graph"].replay()
            else:
                entry["step"]()
            if save_slots is not None and i in save_slots:
                saved[save_slots[i], :share].copy_(st["x"])
        return st["x"].clone()

    def _share(self, frames: torch.Tensor) -> Tuple[torch.Tensor, int]:
        n = frames.shape[0]
        lo, hi = self._local(n)
        return frames[lo:hi].to(self.device, torch.float16), -(-n // self.world_size)

    @torch.no_grad()
    def _device_inversion(self, cond, latent_frames, save_path, batch_size, save_latents, timesteps_to_save):
        inv_coef, _, ts_up_dev, _ = self._device_tables()
        ts_up = [int(t) for t in reversed(self.scheduler.timesteps.tolist())]
        plan = saved_timesteps(ts_up, timesteps_to_save)
        slots = {ts_up.index(t): k for k, t in enumerate(plan)}
        n = latent_frames.shape[0]
        x_share, per = self._share(latent_frames)
        saved = torch.zeros((len(plan), per) + tuple(latent_frames.shape[1:]), dtype=torch.float16, device=self.device)
        self._run_steps(x_share, cond, batch_size, inv_coef, ts_up_dev, slots, saved, self._local(n)[0])
        # one collective after the last step: [G * n_saved, per, ...] -> per saved timestep, the N frames in order
        full = all_gather(saved, self.world_size, self.group, self.comm)
        full = full.view((self.world_size, len(plan), per) + tuple(latent_frames.shape[1:]))
        self._saved = {t: full[:, k].reshape((self.world_size * per,) + tuple(latent_frames.shape[1:]))[:n].clone()
                       for k, t in enumerate(plan)}
        del full, saved
        if save_latents and save_path is not None and self.rank == 0:
            os.makedirs(os.path.join(save_path, "latents"), exist_ok=True)
            for t, v in self._saved.items():
                torch.save(v, os.path.join(save_path, "latents", f"noisy_latents_{t}.pt"))
        return self._saved[plan[-1]].clone()

    @torch.no_grad()
    def _device_sample(self, x, cond, batch_size):
        _, rec_coef, _, ts_dn_dev = self._device_tables()
        x_share, _ = self._share(x)
        return self._gathered(self._run_steps(x_share, cond, batch_size, rec_coef, ts_dn_dev,
                                              frame0=self._local(x.shape[0])[0]), x.shape[0])


def resize_frames(frames_u8: torch.Tensor, size) -> torch.Tensor:
    """uint8 RGB frames [N, H_in, W_in, 3] at their native size -> [N, H, W, 3], size = (H, W) or an int for a square:
    PIL's `Image.resize((W, H), Image.LANCZOS)` of every frame, which is how the reference brings frames to the size
    it edits at.  Its `save_video_frames` resizes every frame to the `--W x --H` it is given (util.py:28; preprocess.py
    recommends 672 x 384 for landscape and 384 x 672 for portrait videos), and its drivers resize square frames to
    512 x 512 (run_tokenflow_pnp.py:174-175, run_tokenflow_sdedit.py:136-137, preprocess.py:191-192).  Sides that
    are multiples of 8 give latents of (H / 8, W / 8); the UNet takes any latent shape.

    CUDA frames are resized on the device by `tf_resize_u8`, bit for bit PIL's result; CPU frames go through PIL
    itself.  An unchanged size returns a copy, as PIL does."""
    h, w = (size, size) if isinstance(size, int) else (int(size[0]), int(size[1]))
    assert frames_u8.dtype == torch.uint8 and frames_u8.dim() == 4 and frames_u8.shape[-1] == 3
    if frames_u8.is_cuda:
        from . import ops as tf_ops
        return tf_ops.default_ops().resize_frames(frames_u8, (h, w))
    import numpy as np
    from PIL import Image
    return torch.from_numpy(np.stack([np.asarray(Image.fromarray(f).resize((w, h), Image.LANCZOS))
                                      for f in frames_u8.contiguous().numpy()]))


def canny_cond(frames_u8: torch.Tensor, low: float = 100, high: float = 200) -> torch.Tensor:
    """uint8 RGB frames [N, H, W, 3] -> the ControlNet conditioning [N, 3, H, W] fp16 of the reference's
    `get_canny_cond` (preprocess.py:113-127): `cv2.Canny(frame, low, high)` of every frame, the edge map stacked
    three times and divided by 255, so every value is 0 or 1.  The reference feeds Canny
    `np.uint8(255 * fp16(ToTensor(frame)))`, which is the frame's own bytes, so the frames `resize_frames` returns
    go in as they are.

    CUDA frames go through `tf_canny_u8` on the device (bit for bit cv2's edges) and come back channels_last, the
    layout the ControlNet's first convolution reads; CPU frames go through `cv2.Canny` itself."""
    assert frames_u8.dtype == torch.uint8 and frames_u8.dim() == 4 and frames_u8.shape[-1] == 3
    if frames_u8.is_cuda:
        from . import ops as tf_ops
        return tf_ops.default_ops().canny(frames_u8, low, high, edges=False)[1]
    import cv2
    import numpy as np
    edges = np.stack([cv2.Canny(f, low, high) for f in frames_u8.contiguous().numpy()])
    image = np.concatenate([edges[..., None]] * 3, axis=-1)
    return torch.from_numpy(image.astype(np.float32) / 255.0).permute(0, 3, 1, 2).to(torch.float16)


def _native_vae(vae) -> bool:
    p = next(vae.parameters())
    return p.is_cuda and p.dtype == torch.float16


@torch.no_grad()
def encode_imgs(vae, frames_u8: torch.Tensor, batch_size: int = 10, deterministic: bool = True,
                generator: Optional[torch.Generator] = None) -> torch.Tensor:
    """uint8 RGB frames [N, H, W, 3] -> scaled latents [N, 4, H/8, W/8] in the VAE's dtype (reference
    preprocess.py:174-182, run_tokenflow_pnp.py:145-153): `2 * ToTensor(frames).to(dtype) - 1`, encoded in batches of
    `batch_size`, the posterior mean (or a sample) times 0.18215.

    A CUDA fp16 VAE gets the uint8 frames on the device and `tf_frames_to_nhwc` computes the encoder input there, bit
    for bit the reference's host conversion, in the channels_last layout (NCHW when the VAE's weights are NCHW).
    Otherwise the conversion is the reference's: an fp32 quotient on the host, then the dtype's ops."""
    from .vae import SCALING_FACTOR
    assert frames_u8.dtype == torch.uint8 and frames_u8.dim() == 4 and frames_u8.shape[-1] == 3
    p = next(vae.parameters())
    if _native_vae(vae):
        from . import ops as tf_ops
        imgs = tf_ops.default_ops().frames_to_nhwc(frames_u8.to(p.device))
        if not vae.encoder.conv_in.weight.is_contiguous(memory_format=torch.channels_last):
            imgs = imgs.contiguous()
    else:
        imgs = frames_u8.cpu().permute(0, 3, 1, 2).contiguous().float().div(255).to(p.dtype).to(p.device)
        imgs = 2 * imgs - 1
    latents = []
    for i in range(0, len(imgs), batch_size):
        posterior = vae.encode(imgs[i:i + batch_size]).latent_dist
        latent = posterior.mean if deterministic else posterior.sample(generator)
        latents.append(latent * SCALING_FACTOR)
    return torch.cat(latents).contiguous()


@torch.no_grad()
def decode_latents(vae, latents: torch.Tensor, batch_size: int = 10) -> torch.Tensor:
    """Scaled latents [N, 4, h, w] -> uint8 RGB frames [N, 8h, 8w, 3] on the latents' device (reference
    preprocess.py:163-172, run_tokenflow_pnp.py:156-163 and the uint8 conversion of util.save_video / ToPILImage):
    `latents / 0.18215` decoded in batches of `batch_size`, then `((img / 2 + 0.5).clamp(0, 1) * 255).to(uint8)`.
    A CUDA fp16 VAE runs that conversion as `tf_nhwc_to_frames`, bit for bit, reading the decoder's channels_last
    output in place."""
    from .vae import SCALING_FACTOR
    native = _native_vae(vae)
    if native:
        from . import ops as tf_ops
        ops = tf_ops.default_ops()
    frames = []
    for b in range(0, latents.shape[0], batch_size):
        imgs = vae.decode(1 / SCALING_FACTOR * latents[b:b + batch_size]).sample
        if native:
            frames.append(ops.nhwc_to_frames(imgs))
        else:
            frames.append(((imgs / 2 + 0.5).clamp(0, 1) * 255).to(torch.uint8).permute(0, 2, 3, 1))
    return torch.cat(frames).contiguous()


def ddim_eps(latents: torch.Tensor, saved: Dict[int, torch.Tensor], scheduler) -> torch.Tensor:
    """The noise that takes the clean latents to the noisiest inverted ones (reference run_tokenflow_pnp.py:186-193):
    `saved` is {t: latents} as `LatentInverter.saved_latents()` returns it (the reference globs the
    noisy_latents_<t>.pt files and takes the largest t), and eps = (x_T - mu_T * x_0) / sigma_T with the scheduler's
    0-dim fp32 alphas, in fp16."""
    noisest = max(int(t) for t in saved)
    noisy = saved[noisest].to(latents.device)
    alpha_prod_T = scheduler.alphas_cumprod[noisest]
    mu_T, sigma_T = alpha_prod_T ** 0.5, (1 - alpha_prod_T) ** 0.5
    eps = (noisy - mu_T * latents) / sigma_T
    return eps.to(torch.float16)


def write_inversion_prompt(save_path: str, prompt: str) -> None:
    """Reference preprocess.py:313-314."""
    os.makedirs(save_path, exist_ok=True)
    with open(os.path.join(save_path, "inversion_prompt.txt"), "w") as f:
        f.write(prompt)
