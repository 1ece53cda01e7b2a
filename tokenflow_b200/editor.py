"""The caller of the hot path: the denoising loop of the reference drivers
(run_tokenflow_pnp.py:195-240, 264-273; run_tokenflow_sdedit.py:154-205), without the parts that
need Stable-Diffusion weights (VAE, CLIP, image/video I/O — out of scope, SURVEY.md §2).

`TokenFlowEditor` is parameterised by the hook module, so the same loop runs
  * this package's hooks (`tokenflow_b200.tokenflow_utils`, CUDA kernels) — the product,
  * the unmodified reference hooks (via oracle/ref_shim.py) — golden-vector generation,
  * this package's hooks with oracle ops installed — CPU plumbing tests / CPU baseline.

Per denoising step (reference batched_denoise_step, :220-233):
  1. draw one random keyframe per batch of B frames (CPU generator, like the reference);
  2. pivotal pass: UNet over [source | uncond | cond] x K keyframes, output discarded — it only
     fills the per-block caches (pivot features, extended-attention outputs);
  3. frame passes: UNet over each batch of B frames; self-attention is replaced by NN propagation;
  4. classifier-free guidance + DDIM update per batch.

With a ControlNet (controlnet.py) and the Canny conditioning of the frames (`preprocess.canny_cond`), every UNet call
is preceded by the ControlNet on the same batch, each sample reading the conditioning of its own frame (a pivotal
sample: its keyframe's), and the UNet adds the residuals: diffusers' ControlNet pipeline without guess_mode, applied
to the source stream as well, as the reference's inversion does.  It composes with either mode.
"""
from __future__ import annotations

import contextlib
import os
from typing import Callable, Dict, Optional

import torch
import torch.nn as nn

from .ops import frame_share, gather_frames


class TokenFlowEditor(nn.Module):
    def __init__(self, unet: nn.Module, scheduler, hooks, config: Dict, text_embeds: torch.Tensor,
                 pnp_guidance_embeds: torch.Tensor, source_latents: Optional[Callable[[int], torch.Tensor]] = None,
                 world_size: int = 1, rank: int = 0, group=None, controlnet: Optional[nn.Module] = None,
                 controlnet_cond: Optional[torch.Tensor] = None):
        """config keys (names follow configs/config_pnp.yaml): n_frames, batch_size, n_timesteps,
        guidance_scale, mode ('pnp' | 'sdedit'), pnp_attn_t, pnp_f_t, start (sdedit), latents_path,
        controlnet_conditioning_scale (default 1.0).
        text_embeds: [2, L, C] (uncond, cond);  pnp_guidance_embeds: [1, L, C] (inversion prompt).
        controlnet, controlnet_cond: an optional ControlNet and the [N, 3, H, W] conditioning of all N frames."""
        super().__init__()
        if (controlnet is None) != (controlnet_cond is None):
            raise ValueError("TokenFlowEditor needs both controlnet and controlnet_cond, or neither")
        # kept out of the module tree: the register_* hooks walk this module's submodules, and the ControlNet's
        # attention must stay the plain one
        object.__setattr__(self, "controlnet", controlnet)
        self.unet = unet
        self.scheduler = scheduler
        self.hooks = hooks
        self.config = dict(config)
        if self.config.get("dual_stream"):
            raise ValueError("config['dual_stream'] is not supported: a step runs as one fused UNet call on one stream "
                             "(config['fused_pass'])")
        if world_size > 1 and not self.config.get("fused_pass", False):
            raise ValueError(f"world_size = {world_size} needs config['fused_pass']: the fused step is the only "
                             "multi-rank schedule")
        self.text_embeds = text_embeds
        self.pnp_guidance_embeds = pnp_guidance_embeds
        self.latents_path = self.config.get("latents_path")
        self._source_latents = source_latents
        self.device = next(unet.parameters()).device
        self.scheduler.set_timesteps(self.config["n_timesteps"], device=self.device)
        if self.config.get("mode", "pnp") == "sdedit":        # run_tokenflow_sdedit.py:57
            start = float(self.config.get("start", 0.9))
            self.scheduler.timesteps = self.scheduler.timesteps[int(1 - start * self.config["n_timesteps"]):]
        self.keyframe_log = []
        self.world_size, self.rank, self.group = world_size, rank, group
        self._src_override = None
        # host ints and device scalars of the timesteps, resolved once: the per-step code never has to read
        # a device tensor back (`int(t)` on a CUDA tensor is a full stream synchronisation)
        self._t_host = [int(t) for t in self.scheduler.timesteps]
        self._t_dev = {t: torch.tensor(t, device=self.device) for t in self._t_host}
        self._t_index = {t: i for i, t in enumerate(self._t_host)}
        # keyframe draws: world_size == 1 follows the reference (global CPU RNG, run_tokenflow_pnp.py:224); with
        # several ranks every rank must draw the SAME keyframes, so the draws come from a dedicated generator
        # seeded identically everywhere (config "keyframe_seed", default = the reference's seed 1) and are
        # independent of whatever else consumes the global RNG on a rank.  config["check_keyframes"] additionally
        # all-gathers the draw and asserts equality (debug / verify runs).
        self._kf_gen = None
        if world_size > 1 or "keyframe_seed" in self.config:
            self._kf_gen = torch.Generator().manual_seed(int(self.config.get("keyframe_seed", self.config.get("seed", 1))))
        self.comm = None                      # ops.Communicator (C-ABI NCCL all-gather), see attach_communicator
        # DDIM coefficients per schedule position, on the device, for the fused CFG+DDIM kernel:
        # sqrt(1-a_t), 1/sqrt(a_t), sqrt(a_prev), sqrt(1-a_prev) as the fp32 values the eager expression uses
        # (a v-prediction scheduler: sqrt(a_t), sqrt(1-a_t), sqrt(a_prev), sqrt(1-a_prev))
        self._coef_table = self._make_coef_table()
        self._graphs = {}                     # injection variant -> captured step
        self._graph_pool = None
        self._g_static = None
        self._text_cache = {}
        self._shard_cache = {}
        self._ccond = None
        if controlnet is not None:
            cl = next(controlnet.parameters()).is_contiguous(memory_format=torch.channels_last)
            self._ccond = controlnet_cond.to(self.device, next(controlnet.parameters()).dtype).contiguous(
                memory_format=torch.channels_last if cl else torch.contiguous_format)

    def _residuals(self, latent_model_input, t, text, cond):
        """UNet keyword arguments of one call: the ControlNet's residuals for `cond`, or {} without a ControlNet."""
        from .controlnet import controlnet_residuals
        return controlnet_residuals(self.controlnet, latent_model_input, t, text, cond,
                                    float(self.config.get("controlnet_conditioning_scale", 1.0)))

    # ------------------------------------------------------------------------------------
    def init_method(self):
        """run_tokenflow_pnp.py:235-240 / run_tokenflow_sdedit.py:191-193."""
        h = self.hooks
        if self.config.get("mode", "pnp") == "pnp":
            n = self.config["n_timesteps"]
            qk_t = int(n * self.config.get("pnp_attn_t", 0.5))
            conv_t = int(n * self.config.get("pnp_f_t", 0.8))
            self.qk_injection_timesteps = self.scheduler.timesteps[:qk_t] if qk_t >= 0 else []
            self.conv_injection_timesteps = self.scheduler.timesteps[:conv_t] if conv_t >= 0 else []
            h.register_extended_attention_pnp(self, self.qk_injection_timesteps)
            h.register_conv_injection(self, self.conv_injection_timesteps)
        else:
            h.register_extended_attention(self)
        h.set_tokenflow(self.unet)

    def source_latents_t(self, t: int) -> torch.Tensor:
        if self._src_override is not None and self._src_override[0] == int(t):
            return self._src_override[1]
        if self._source_latents is not None:
            return self._source_latents(t)
        return self.hooks.load_source_latents_t(t, self.latents_path)

    # ------------------------------------------------------------------------------------
    @torch.no_grad()
    def denoise_step(self, x, t, indices):
        """run_tokenflow_pnp.py:195-218."""
        source_latents = self.source_latents_t(int(t))[indices].to(x.device, x.dtype)
        latent_model_input = torch.cat([source_latents] + ([x] * 2))
        self.hooks.register_time(self, int(t))
        text_embed_input = torch.cat([self.pnp_guidance_embeds.repeat(len(indices), 1, 1),
                                      torch.repeat_interleave(self.text_embeds, len(indices), dim=0)])
        res = {}
        if self.controlnet is not None:
            c = self._ccond[indices.to(self._ccond.device)]
            res = self._residuals(latent_model_input, t, text_embed_input, torch.cat([c, c, c]))
        noise_pred = self.unet(latent_model_input, t, encoder_hidden_states=text_embed_input, **res)['sample']
        _, noise_pred_uncond, noise_pred_cond = noise_pred.chunk(3)
        noise_pred = noise_pred_uncond + self.config["guidance_scale"] * (noise_pred_cond - noise_pred_uncond)
        return self.scheduler.step(noise_pred, t, x)['prev_sample']

    def _autocast(self):
        if self.device.type == "cuda" and self.config.get("autocast", True):
            return torch.autocast(device_type="cuda", dtype=torch.float16)    # run_tokenflow_pnp.py:220
        return contextlib.nullcontext()

    def draw_keyframes(self, n: int) -> torch.Tensor:
        """run_tokenflow_pnp.py:224 — one uniformly random frame inside every batch (CPU RNG).  A last batch of
        r = n mod B frames gets its keyframe from one more draw, randint(r), after the full batches' draws: when B
        divides n the draws are the reference's, and no frame is dropped when it does not (the reference truncates
        n to a multiple of B, run_tokenflow_pnp.py:121-123)."""
        batch_size = self.config["batch_size"]
        full, rest = divmod(n, batch_size)
        gen = {} if self._kf_gen is None else {"generator": self._kf_gen}
        idx = torch.randint(batch_size, (full,), **gen) + torch.arange(0, full * batch_size, batch_size)
        if rest:
            idx = torch.cat([idx, torch.randint(rest, (1,), **gen) + full * batch_size])
        if self.world_size > 1 and self.config.get("check_keyframes", False):
            import torch.distributed as dist
            mine = idx.to(self.device if dist.get_backend(self.group) == "nccl" else "cpu")
            everyone = [torch.empty_like(mine) for _ in range(self.world_size)]
            dist.all_gather(everyone, mine, group=self.group)
            for r_, other in enumerate(everyone):
                if not torch.equal(other.cpu(), idx):
                    raise RuntimeError(f"rank {self.rank} drew keyframes {idx.tolist()} but rank {r_} drew "
                                       f"{other.cpu().tolist()}: the ranks' keyframe generators are out of step")
        return idx

    def _make_coef_table(self):
        import numpy as np
        sch, rows = self.scheduler, []
        ratio = sch.num_train_timesteps // sch.num_inference_steps
        for t in self._t_host:
            a_t = float(sch._alpha(t))
            a_prev = float(sch._alpha(t - ratio))
            if sch.prediction_type == "v_prediction":
                # tf_cfg_ddim_v: the step multiplies by the Python floats below, which ATen rounds to fp32
                rows.append([float(np.float32(v)) for v in (a_t ** 0.5, (1 - a_t) ** 0.5, a_prev ** 0.5,
                                                             (1 - a_prev) ** 0.5)])
                continue
            # the step divides the fp16 latents by the Python float sqrt(a_t): ATen multiplies by the reciprocal taken in
            # double and rounded to fp32, which is not always the fp32 reciprocal of the fp32 sqrt (50 steps: 8 rows)
            s1 = np.float32((1 - a_t) ** 0.5)
            rows.append([float(s1), float(np.float32(1.0 / a_t ** 0.5)), float(np.float32(a_prev ** 0.5)),
                         float(np.float32((1 - a_prev) ** 0.5))])
        return torch.tensor(rows, dtype=torch.float32, device=self.device)

    def attach_communicator(self, comm):
        """Route the pivotal pass's all-gathers through the C ABI (tf_allgather) instead of torch.distributed."""
        self.comm = comm

    def batched_denoise_step(self, x, t, indices):
        """run_tokenflow_pnp.py:220-233.  With config["fused_pass"] the pivotal samples and the frame samples go
        through the UNet in ONE call (the keyframe caches a block fills from the first part of the batch are consumed
        by the second part inside the same block) — identical arithmetic, half the kernel launches; this is also the
        only multi-rank form.  Otherwise the reference's schedule on one rank: the pivotal pass, then a frame pass per
        batch or per config["frames_per_pass"] frames."""
        if self.config.get("fused_pass", False):
            with self._autocast():
                return self._fused_step(x, t, indices)
        h = self.hooks
        batch_size = self.config["batch_size"]
        with self._autocast():
            pivotal_idx = self.draw_keyframes(len(x))
            self.keyframe_log.append(pivotal_idx.tolist())
            h.register_pivotal(self, True)
            self.denoise_step(x[pivotal_idx], t, indices[pivotal_idx])
            h.register_pivotal(self, False)
            per_pass = int(self.config.get("frames_per_pass", batch_size))
            if per_pass == batch_size:                                   # the reference's schedule (:229-231)
                denoised = []
                for i, b in enumerate(range(0, len(x), batch_size)):
                    if b + batch_size <= len(x):
                        h.register_batch_idx(self, i)
                    else:
                        # a short last batch: the reference's per-batch weights would place its frames as if the
                        # batch had len(x) - b frames (tokenflow_utils.py:375-378); the table keeps the stride B
                        h.register_frame_table(self, *self.frame_table(list(range(b, len(x)))))
                    denoised.append(self.denoise_step(x[b:b + batch_size], t, indices[b:b + batch_size]))
                return torch.cat(denoised)
            # same arithmetic, fewer and larger UNet passes: frames of several batches in one pass, each frame
            # carrying its own (keyframe, previous keyframe, weight) — the per-frame table the kernels take
            denoised = []
            for b in range(0, len(x), per_pass):
                frames = list(range(b, min(len(x), b + per_pass)))
                h.register_frame_table(self, *self.frame_table(frames))
                denoised.append(self.denoise_step(x[b:b + per_pass], t, indices[b:b + per_pass]))
            return torch.cat(denoised)

    def frame_table(self, frames):
        """Per-frame (keyframe, previous keyframe, blend weight) for global frame ids — the reference's
        batch_idx arithmetic (tokenflow_utils.py:331-333, :375-383) evaluated per frame.  The frames of a short last
        batch keep the nominal stride B, so frame g blends with weight blend_weights(B)[g % B]; the reference's hooks,
        given a short batch of r frames, would compute their positions with n_frames = r (:312, :375-378)."""
        from .ops import blend_weights
        B = self.config["batch_size"]
        w = blend_weights(B)
        kf_a = [g // B for g in frames]
        kf_b = [(g // B) - 1 if g >= B else -1 for g in frames]
        return kf_a, kf_b, [w[g % B] for g in frames]

    def _timestep_pair(self, t):
        """(host int, device scalar) of a timestep without reading the device when `t` is a host value."""
        t_int = t if isinstance(t, int) else int(t)
        t_dev = self._t_dev.get(t_int)
        if t_dev is None:
            t_dev = self._t_dev[t_int] = torch.tensor(t_int, device=self.device)
        return t_int, t_dev

    def step_index(self, x, i: int, indices=None):
        """Denoising step number `i` of the schedule, addressed by index so that no device value is read
        back on the host (the reference's loop passes a CUDA 0-dim timestep, which costs a stream
        synchronisation per use)."""
        if indices is None:
            indices = torch.arange(len(x))
        return self.batched_denoise_step(x, self._t_host[i % len(self._t_host)], indices)

    # ------------------------------------------------------------------------------------
    # fused step: ONE UNet call per denoising step and rank, [pivotal samples | this rank's frames x 3 streams]
    # ------------------------------------------------------------------------------------
    def _pivotal_slots(self, K: int):
        """(stream, keyframe) of every pivotal sample this rank runs, in batch order.  One rank: the reference's
        [src | uncond | cond] x K batch.  Several ranks: this rank's m = ceil(3K/G) slots of that order (the tail is
        padded with repeats of the last sample, whose results are ignored)."""
        G, r = self.world_size, self.rank
        if G == 1:
            return [divmod(i, K) for i in range(3 * K)], None
        key = (K, id(self.comm))
        shard = self._shard_cache.get(key)
        if shard is None:                     # one shard context per (K, communicator): it caches device index tensors
            shard = self._shard_cache[key] = self.hooks.PivotalShard(G, r, K, self.group, comm=self.comm)
        return [divmod(min(i, 3 * K - 1), K) for i in shard.slots], shard

    def _fused_text(self, slots, per):
        """Text embeddings of a call over the pivotal `slots` (none for a later frame chunk) and `per` frames."""
        key = (tuple(slots), per)
        text = self._text_cache.get(key)
        if text is None:
            emb = [self.pnp_guidance_embeds[0] if s_ == 0 else self.text_embeds[s_ - 1] for s_, _ in slots]
            text = torch.cat(([torch.stack(emb)] if emb else []) + [self.pnp_guidance_embeds.repeat(per, 1, 1),
                             torch.repeat_interleave(self.text_embeds, per, dim=0)])
            if len(self._text_cache) >= 3:        # a step makes at most three: pivotal + chunk 0, chunk, last chunk
                self._text_cache = {}
            self._text_cache[key] = text
        return text

    def _rank_frames(self, N: int):
        """Frames [lo, hi) this rank edits (`ops.frame_share`, the inversion stage's split)."""
        G, per = self.world_size, -(-N // self.world_size)
        if (G - 1) * per >= N:
            raise ValueError(f"{N} frames in shares of {per} leave rank {G - 1} of {G} without frames: use fewer "
                             "ranks or more frames")
        return frame_share(N, G, self.rank)

    def _frame_chunks(self, lo: int, hi: int):
        """[a, b) frame ranges of the rank's UNet calls: chunks of at most config["frames_per_pass"] frames, or one."""
        c = int(self.config.get("frames_per_pass", hi - lo))
        if c < 1:
            raise ValueError(f"config['frames_per_pass'] = {c}: a UNet call needs at least one frame")
        return [(a, min(hi, a + c)) for a in range(lo, hi, c)]

    def _fused_compute(self, x, src_all, piv_idx, t_dev, t_int, coef, slots, shard):
        """Device work of one fused step.  Everything that varies from step to step arrives in device tensors
        (`piv_idx`: which latents are the pivotal samples, `t_dev`, `coef`: the DDIM coefficients), so the same
        function body can be captured once into a CUDA graph and replayed (run_tokenflow_pnp.py:195-233)."""
        h, G = self.hooks, self.world_size
        N = x.shape[0]
        lo, hi = self._rank_frames(N)
        chunks = self._frame_chunks(lo, hi)
        piv_lat = torch.cat([src_all, x]).index_select(0, piv_idx)       # slot (s, f): src[kf_f] if s == 0 else x[kf_f]
        c_piv = None
        if self.controlnet is not None:
            # the same gather as the pivotal latents (index f or N + f: keyframe f), so a graph replay stays sync-free
            c_piv = self._ccond.index_select(0, piv_idx.remainder(N))
        h.register_time(self, t_int)
        h.register_pivotal(self, False)
        x_local = None if len(chunks) == 1 else x.new_empty((hi - lo,) + tuple(x.shape[1:]))
        for j, (a, b) in enumerate(chunks):
            # the first call also carries the pivotal samples and fills every block's keyframe caches; a later chunk is
            # a plain frame pass over [a, b) that reads them from the modules (kf_attn_output, _tf_pivot_unit)
            piv = (piv_lat,) if j == 0 else ()
            n_piv = len(slots) if j == 0 else 0
            xs, srcs = x[a:b], src_all[a:b]
            latent_model_input = torch.cat(piv + (srcs, xs, xs))
            text = self._fused_text(slots if j == 0 else (), b - a)
            res = {}
            if c_piv is not None:
                c_loc = self._ccond[a:b]
                res = self._residuals(latent_model_input, t_dev, text,
                                      torch.cat(((c_piv,) if j == 0 else ()) + (c_loc, c_loc, c_loc)))
            h.register_shard(self, shard if j == 0 else None)
            h.register_frame_table(self, *self.frame_table(list(range(a, b))))
            h.register_fused(self, n_piv)
            try:
                noise_pred = self.unet(latent_model_input, t_dev, encoder_hidden_states=text, **res)['sample'][n_piv:]
            finally:
                h.register_fused(self, 0)
                h.register_shard(self, None)
            # classifier-free guidance + DDIM update of the chunk's frames, into its slice of this rank's output
            out = None if x_local is None else x_local[a - lo:b - lo]
            _, npu, npc = noise_pred.chunk(3)
            ops = self._cuda_ops()
            if ops is not None and coef is not None and npu.dtype == torch.float16 and xs.dtype == torch.float16:
                step = ops.cfg_ddim_v if self.scheduler.prediction_type == "v_prediction" else ops.cfg_ddim
                y = step(npu, npc, xs, coef, self.config["guidance_scale"], out=out)    # one kernel, same roundings
            else:
                noise_pred = npu + self.config["guidance_scale"] * (npc - npu)
                y = self.scheduler.step(noise_pred, t_int, xs)['prev_sample'].contiguous()
                if out is not None:
                    out.copy_(y)
            if x_local is None:
                x_local = y
        # one all-gather of every rank's frames
        return gather_frames(x_local, N, G, self.group, self.comm)

    def _cuda_ops(self):
        """The CUDA op object if the hooks run on it (None under the oracle test seam / on CPU)."""
        if self.device.type != "cuda":
            return None
        ops = self.hooks._ops() if hasattr(self.hooks, "_ops") else None
        return ops if hasattr(ops, "cfg_ddim") else None

    def _piv_index_list(self, kf_list, slots, N):
        return [kf_list[f_] if s_ == 0 else N + kf_list[f_] for s_, f_ in slots]

    def _variant(self, t_int):
        """Which hooks inject at this timestep — the only way `t` changes the captured kernel sequence."""
        if self.config.get("mode", "pnp") != "pnp":
            return (False, False)
        qk = {int(v) for v in (self.qk_injection_timesteps.tolist() if torch.is_tensor(self.qk_injection_timesteps)
                               else self.qk_injection_timesteps)}
        conv = {int(v) for v in (self.conv_injection_timesteps.tolist() if torch.is_tensor(self.conv_injection_timesteps)
                                 else self.conv_injection_timesteps)}
        return (t_int in qk or t_int == 1000, t_int in conv or t_int == 1000)

    @torch.no_grad()
    def _fused_step(self, x, t, indices):
        """One UNet call per denoising step and rank: [pivotal samples | this rank's frames x 3 streams]."""
        N, B = len(x), self.config["batch_size"]
        K = -(-N // B)                                        # a last keyframe group may be short
        self._rank_frames(N)                                  # refuses a split that leaves a rank without frames
        t_int, t_dev = self._timestep_pair(t)
        pivotal_idx = self.draw_keyframes(N)
        kf_list = pivotal_idx.tolist()
        self.keyframe_log.append(kf_list)
        src_all = self.source_latents_t(t_int)
        if not (indices.device.type == "cpu" and indices.numel() == src_all.shape[0]
                and torch.equal(indices, torch.arange(indices.numel()))):
            src_all = src_all[indices]                        # (identity in the drivers: all frames, in order)
        src_all = src_all.to(x.device, x.dtype)
        slots, shard = self._pivotal_slots(K)
        idx_host = torch.tensor(self._piv_index_list(kf_list, slots, N), dtype=torch.int64)
        i = self._t_index.get(t_int)
        coef = self._coef_table[i] if i is not None else None
        if self.config.get("cuda_graph", False) and self.device.type == "cuda" and coef is not None:
            return self._graph_replay(x, src_all, idx_host, t_int, i, slots, shard)
        piv_idx = idx_host.to(x.device, non_blocking=True) if x.is_cuda else idx_host
        return self._fused_compute(x, src_all, piv_idx, t_dev, t_int, coef, slots, shard)

    # ------------------------------------------------------------------------------------
    # CUDA graphs (SURVEY.md §8 f-2): the fused step's shape is static, so it is captured once per injection
    # variant (PnP: q/k + conv injection, conv injection only, none) and replayed.  Per replay the host only
    # refreshes five small static inputs: latents, source latents, the pivotal gather index, the timestep and
    # the DDIM coefficients.  TMA descriptors, frame tables and attention tables are kernel parameters baked at
    # capture; NCCL all-gathers are captured in-graph.
    # ------------------------------------------------------------------------------------
    def _graph_replay(self, x, src_all, idx_host, t_int, i, slots, shard):
        variant = self._variant(t_int)
        st = self._g_static
        if st is None or st["x"].shape != x.shape or st["x"].dtype != x.dtype:
            st = self._g_static = {
                "x": torch.empty_like(x), "src": torch.empty_like(x),
                "idx": torch.zeros(len(idx_host), dtype=torch.int64, device=x.device),
                "t": torch.zeros((), dtype=torch.int64, device=x.device),
                "coef": torch.zeros(4, dtype=torch.float32, device=x.device)}
            self._graphs = {}
        if x.data_ptr() != st["x"].data_ptr():
            st["x"].copy_(x, non_blocking=True)
        if src_all.data_ptr() != st["src"].data_ptr():
            st["src"].copy_(src_all, non_blocking=True)
        st["idx"].copy_(idx_host.pin_memory(), non_blocking=True)
        st["t"].copy_(self._t_dev[t_int], non_blocking=True)
        st["coef"].copy_(self._coef_table[i], non_blocking=True)
        entry = self._graphs.get(variant)
        if entry is None:
            entry = self._graphs[variant] = self._capture(st, t_int, slots, shard)
        entry["graph"].replay()
        entry["replays"] += 1
        return entry["out"].clone()

    def _capture(self, st, t_int, slots, shard):
        ops = self._cuda_ops()
        run = lambda: self._fused_compute(st["x"], st["src"], st["idx"], st["t"], t_int, st["coef"], slots, shard)
        # warm-up on a side stream (cuDNN autotuning, lazy initialisation, allocator growth) — not captured
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        saved_timing = ops._timing if ops is not None else None
        if ops is not None:
            ops._timing = None
        with torch.cuda.stream(side):
            for _ in range(int(self.config.get("graph_warmup", 2))):
                run()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        events = [] if saved_timing is not None else None
        launches0 = ops.launch_count() if ops is not None else 0
        if ops is not None:
            ops._timing = events                # per-launch EXTERNAL events recorded as graph nodes
        try:
            with torch.cuda.graph(graph, pool=self._graph_pool, capture_error_mode="thread_local"):
                out = run()
        finally:
            if ops is not None:
                ops._timing = saved_timing
        if self._graph_pool is None:
            self._graph_pool = graph.pool()
        return {"graph": graph, "out": out, "events": events, "replays": 0,
                "launches": (ops.launch_count() - launches0) if ops is not None else 0}

    def graph_launches_per_step(self) -> int:
        """Kernels of this library inside one replay of the most recently used step graph."""
        used = [e for e in self._graphs.values() if e["replays"]]
        return max((e["launches"] for e in used), default=0)

    def mark_graph_replays(self):
        """Start of a measured region: `graph_kernel_times(since_mark=True)` then covers the replays after this call."""
        for entry in self._graphs.values():
            entry["mark"] = entry["replays"]

    @staticmethod
    def aggregate_graph_events(entries, since_mark=False):
        """{kernel: {"launches", "ms", "work"}} over the replays of the captured step graphs.  The event nodes are part
        of a graph and every replay overwrites their timestamps, so what can be read is the LAST replay of each
        variant; a variant that was replayed n times contributes n times its last replay.  Returns (totals, steps)."""
        agg, steps = {}, 0
        for entry in entries:
            n = entry["replays"] - (entry.get("mark", 0) if since_mark else 0)
            if n <= 0 or not entry.get("events"):
                continue
            steps += n
            for name, work, s_, e_ in entry["events"]:
                a = agg.setdefault(name, {"launches": 0, "ms": 0.0, "work": 0.0})
                a["launches"] += n
                a["ms"] += n * s_.elapsed_time(e_)
                a["work"] += n * work
        return agg, steps

    def graph_kernel_times(self, since_mark=False):
        """Per-kernel totals of the step graphs' per-launch event nodes (see `aggregate_graph_events`)."""
        torch.cuda.synchronize()
        return self.aggregate_graph_events(self._graphs.values(), since_mark)

    # ------------------------------------------------------------------------------------
    # host-buffer entry point (bench `e2e`): latents live in pinned host memory
    # ------------------------------------------------------------------------------------
    def edit_step_host(self, x_host: torch.Tensor, src_host_t: torch.Tensor, t: int, out_host: torch.Tensor):
        """One denoising step with HOST latents: H2D of this step's noisy latents and source latents,
        the step, D2H of the denoised latents, stream-synchronised before returning."""
        x = x_host.to(self.device, non_blocking=True)
        self._src_override = (int(t), src_host_t.to(self.device, non_blocking=True))
        try:
            y = self.batched_denoise_step(x, int(t), torch.arange(len(x_host)))
        finally:
            self._src_override = None
        out_host.copy_(y, non_blocking=True)
        if self.device.type == "cuda":
            torch.cuda.current_stream().synchronize()
        return out_host

    def sample_loop(self, x, indices=None, on_step: Optional[Callable] = None):
        """run_tokenflow_pnp.py:264-273 without the VAE decode."""
        if indices is None:
            indices = torch.arange(len(x))
        for i, t in enumerate(self._t_host):          # host ints: nothing is read back from the device per step
            x = self.batched_denoise_step(x, t, indices)
            if on_step is not None:
                on_step(i, t, x)
        return x


# --------------------------------------------------------------------------------------------
# synthetic inputs (SURVEY.md §8d): no SD weights / VAE / CLIP exist here
# --------------------------------------------------------------------------------------------
def synthetic_inputs(n_frames: int, latent_size, ctx_dim: int, n_timesteps: int, seed: int = 1,
                     device="cpu", dtype=torch.float32, ctx_len: int = 77):
    """x ~ N(0,1) [N,4,h,w] (`latent_size` is h = w, or an (h, w) pair); one source latent tensor per sampling
    timestep; text embeddings ~ N(0,1).  Deterministic in `seed` and independent of device."""
    h, w = (latent_size, latent_size) if isinstance(latent_size, int) else tuple(latent_size)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n_frames, 4, h, w, generator=g)
    text = torch.randn(2, ctx_len, ctx_dim, generator=g)
    pnp = torch.randn(1, ctx_len, ctx_dim, generator=g)
    ratio = 1000 // n_timesteps
    timesteps = [(n_timesteps - 1 - i) * ratio + 1 for i in range(n_timesteps)]
    src = {t: torch.randn(n_frames, 4, h, w, generator=g) for t in timesteps}
    conv = lambda z: z.to(device=device, dtype=dtype)
    return conv(x), conv(text), conv(pnp), {t: conv(v) for t, v in src.items()}


def write_latents_dir(path: str, src: Dict[int, torch.Tensor], prompt: str = "synthetic") -> str:
    """The preprocess -> edit hand-off format (preprocess.py:227-229, :313-314):
    <path>/latents/noisy_latents_<t>.pt + <path>/inversion_prompt.txt."""
    lat = os.path.join(path, "latents")
    os.makedirs(lat, exist_ok=True)
    for t, v in src.items():
        torch.save(v, os.path.join(lat, f"noisy_latents_{t}.pt"))
    with open(os.path.join(path, "inversion_prompt.txt"), "w") as f:
        f.write(prompt)
    return lat
