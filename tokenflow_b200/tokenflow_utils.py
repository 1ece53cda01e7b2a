"""Drop-in replacement for the reference's `tokenflow_utils.py` hook layer.

Same public names, signatures and module-state contract as omerbt/TokenFlow's tokenflow_utils.py
(consumed by `from tokenflow_utils import *` in run_tokenflow_pnp.py:16 / run_tokenflow_sdedit.py:15),
so the reference drivers run unchanged — but the three hot operations underneath are hand-written
sm_90a CUDA kernels reached through the C ABI in include/tokenflow_b200.h:

    extended attention      attn1 closure        -> tf_ext_attn_fwd      (reference :114-199, :224-281)
    NN field                TokenFlowBlock       -> tf_unit_rows + tf_nn_field   (:329-348, util.py:61-69)
    propagation             TokenFlowBlock       -> tf_propagate         (:361-397)

There is no PyTorch/CPU fallback: the first hot-path call constructs `ops.CudaOps`, which raises if
the library or an H100 is missing.

Differences from the reference that do not change results:
  * per-pass host work is O(#blocks): module lists are discovered once per model instead of walking
    `named_modules()` of UNet+VAE+CLIP on every register_* call (reference :8,:14);
  * `t in injection_schedule` is a host-side set lookup, not a CUDA-tensor membership test with a
    device sync per attn1 call (reference :124);
  * PnP q/k injection (:124-130) copies nothing — the kernel reads the source stream's q/k;
  * the frame pass can be driven per frame (`register_frame_table`) so frames, not only whole
    batches, shard across GPUs (SURVEY.md §8e); `register_batch_idx` keeps the reference meaning;
  * the pivotal pass can be sharded over GPUs (`PivotalShard`, `register_shard`): per block, one
    all-gather of the packed [q | k | v | pivot unit rows], the extended attention of every sample
    for this rank's query rows (tf_ext_attn_fwd_rows), one all-gather of the attention output.
"""
from __future__ import annotations

import os
import weakref
from typing import List, Optional, Sequence, Type

import torch

from . import ops as tf_ops
from .sd_unet import norm_act
from .util import isinstance_str, batch_cosine_sim  # noqa: F401  (re-exported like the reference)

__all__ = [
    "register_pivotal", "register_batch_idx", "register_frame_table", "register_shard", "register_fused",
    "PivotalShard", "set_strict_dtype",
    "register_time", "load_source_latents_t",
    "register_conv_injection", "register_extended_attention_pnp", "register_extended_attention",
    "make_tokenflow_attention_block", "set_tokenflow", "isinstance_str", "batch_cosine_sim",
]

# --------------------------------------------------------------------------------------------
# operator object (product: CudaOps; tests may install an oracle-backed stand-in)
# --------------------------------------------------------------------------------------------
_OPS = None


def _ops():
    global _OPS
    if _OPS is None:
        from .ops import default_ops
        _OPS = default_ops()        # raises without the .so or without an H100: no fallback
    return _OPS


def _install_ops_for_testing(ops) -> None:
    """Test seam: `tests/` may substitute an op object built on `oracle/` to exercise the hook
    plumbing on CPU.  Pass None to restore the product path."""
    global _OPS
    _OPS = ops


_STRICT_DTYPE = None


def set_strict_dtype(flag) -> None:
    """True: the blended frame-pass output is fp32 like the reference's promoted dtype (:385-388); False: fp16
    (half the HBM write, same values to fp16 rounding); None: follow TOKENFLOW_B200_STRICT_DTYPE (default off)."""
    global _STRICT_DTYPE
    _STRICT_DTYPE = None if flag is None else bool(flag)


def _strict_dtype() -> bool:
    if _STRICT_DTYPE is not None:
        return _STRICT_DTYPE
    return os.environ.get("TOKENFLOW_B200_STRICT_DTYPE", "0") == "1"


# --------------------------------------------------------------------------------------------
# module discovery (cached)
# --------------------------------------------------------------------------------------------
_BLOCK_CACHE: "weakref.WeakKeyDictionary[torch.nn.Module, List[torch.nn.Module]]" = weakref.WeakKeyDictionary()


def _transformer_blocks(root: torch.nn.Module) -> List[torch.nn.Module]:
    blocks = _BLOCK_CACHE.get(root)
    if blocks is None:
        blocks = [m for _, m in root.named_modules() if isinstance_str(m, "BasicTransformerBlock")]
        _BLOCK_CACHE[root] = blocks
    return blocks


def _invalidate_cache(root: Optional[torch.nn.Module] = None) -> None:
    if root is None:
        _BLOCK_CACHE.clear()
    else:
        _BLOCK_CACHE.pop(root, None)


def register_pivotal(diffusion_model, is_pivotal):
    """Reference :7-11."""
    for module in _transformer_blocks(diffusion_model):
        module.pivotal_pass = is_pivotal


def register_batch_idx(diffusion_model, batch_idx):
    """Reference :13-17.  Frame f of the batch uses keyframes (batch_idx, batch_idx-1)."""
    for module in _transformer_blocks(diffusion_model):
        module.batch_idx = batch_idx
        module._tf_frame_table = None


def register_frame_table(diffusion_model, kf_a: Sequence[int], kf_b: Sequence[int], w: Sequence[float]):
    """Extension for frame-granular sharding: per-frame (keyframe, previous keyframe or -1, blend
    weight) for the frames of the next frame pass, replacing the scalar batch_idx."""
    table = (tuple(int(a) for a in kf_a), tuple(int(b) for b in kf_b), tuple(float(x) for x in w))
    for module in _transformer_blocks(diffusion_model):
        module._tf_frame_table = table


class PivotalShard:
    """Multi-GPU pivotal pass (SURVEY.md §8e).  The 3K (stream, keyframe) samples of the pass, in the
    reference's batch order i = stream*K + keyframe, are dealt to the G ranks in contiguous groups of
    m = ceil(3K/G) slots (the tail is padded with dummy samples); an all-gather along that axis
    therefore reproduces the reference's [3K, S, dim] layout in its first 3K slabs.  The extended
    attention is split by query rows (`row_split`): every rank evaluates all 3K samples for its rows,
    which balances the work exactly and keeps q/k-injected sample pairs together.  Collectives go
    through `ops.all_gather` (tf_allgather when a Communicator is attached, else torch.distributed:
    NCCL over NVLink on GPUs, gloo in the CPU tests)."""

    def __init__(self, world_size: int, rank: int, n_keyframes: int, group=None, comm=None):
        self.world_size, self.rank, self.K, self.group = world_size, rank, n_keyframes, group
        self.comm = comm                      # ops.Communicator (tf_allgather through the C ABI) or None
        self.m = -(-3 * n_keyframes // world_size)
        self.slots = list(range(rank * self.m, (rank + 1) * self.m))     # global sample ids (>= 3K: padding)
        self._src_index = {}

    def source_index(self, device) -> torch.Tensor:
        """For each local slot, the global slot of the SOURCE-stream sample of the same keyframe (padding slots map
        to themselves) — the gather index of the PnP conv injection (reference :86-91).  Built once per device and
        kept (a CUDA-graph capture must not create host tensors)."""
        key = str(device)
        idx = self._src_index.get(key)
        if idx is None:
            idx = torch.tensor([i % self.K if i < 3 * self.K else i for i in self.slots], dtype=torch.int64).to(device)
            self._src_index[key] = idx
        return idx

    def all_gather(self, t: torch.Tensor) -> torch.Tensor:
        return tf_ops.all_gather(t, self.world_size, self.group, self.comm)

    def row_split(self, S: int):
        """Query-token range [row0, row0 + nrows) of this rank when the extended attention of ALL 3K samples is
        split by query rows (128-row tiles dealt evenly; trailing ranks may get rows past S = no work)."""
        tiles = -(-S // 128)
        nrows = -(-tiles // self.world_size) * 128
        return self.rank * nrows, nrows

    def global_attention_table(self, inject: bool):
        """(q slab, first k slab, first v slab, key slabs) of all 3K samples in global slab coordinates
        (reference :124-138): what every rank evaluates for its query rows after the q/k/v all-gather."""
        K, tab = self.K, []
        for i in range(3 * K):
            s, f = divmod(i, K)
            if s == 0:
                tab.append((i, i, i, 1))
            else:
                tab.append((f if inject else i, 0 if inject else s * K, s * K, K))
        return tab

    def local_index(self, device) -> torch.Tensor:
        """Global sample id of every local slot (padding slots repeat the last sample), as a device index."""
        key = "local:" + str(device)
        idx = self._src_index.get(key)
        if idx is None:
            idx = torch.tensor([min(i, 3 * self.K - 1) for i in self.slots], dtype=torch.int64).to(device)
            self._src_index[key] = idx
        return idx


def _conv_injection_site(diffusion_model):
    """`up_blocks[1].resnets[1]` (reference :21, :102) whether the caller passes the wrapper (`.unet`) or the
    UNet itself.  A model whose conv-injection hook is installed but whose site cannot be found is an error:
    the fused / sharded batch layouts would otherwise be injected as naive thirds, silently."""
    unet = getattr(diffusion_model, "unet", diffusion_model)
    try:
        return unet.up_blocks[1].resnets[1]
    except (AttributeError, IndexError, TypeError):
        for _, m in diffusion_model.named_modules():
            if getattr(m, "injection_schedule", None) is not None and isinstance_str(m, "ResnetBlock2D"):
                raise RuntimeError("tokenflow_b200: a conv-injection hook is registered but up_blocks[1].resnets[1] "
                                   "cannot be reached from the module passed to register_fused / register_shard")
        return None


def register_fused(diffusion_model, n_pivotal: int):
    """Fused pass: the next UNet call carries `n_pivotal` pivotal samples followed by the frame samples
    ([source | uncond | cond] thirds).  0 restores the reference's separate passes."""
    for module in _transformer_blocks(diffusion_model):
        module._tf_fused = int(n_pivotal)
    res = _conv_injection_site(diffusion_model)
    if res is not None:
        res._tf_fused = int(n_pivotal)


def register_shard(diffusion_model, shard: Optional[PivotalShard]):
    """Install (or clear, with None) the multi-GPU pivotal-pass context on every TokenFlow block."""
    for module in _transformer_blocks(diffusion_model):
        module._tf_shard = shard
        module.attn1._tf_shard = shard
    res = _conv_injection_site(diffusion_model)
    if res is not None:
        res._tf_shard = shard                                # PnP conv-feature injection site


_ATTN_SITES_CACHE: "weakref.WeakKeyDictionary[torch.nn.Module, list]" = weakref.WeakKeyDictionary()


def _timed_modules(unet) -> list:
    """The fixed SD topology the reference hard-codes (:20-40)."""
    mods = _ATTN_SITES_CACHE.get(unet)
    if mods is None:
        mods = [unet.up_blocks[1].resnets[1]]
        for res in (1, 2, 3):
            for block in (0, 1, 2):
                tb = unet.up_blocks[res].attentions[block].transformer_blocks[0]
                mods += [tb.attn1, tb.attn2]
        for res in (0, 1, 2):
            for block in (0, 1):
                tb = unet.down_blocks[res].attentions[block].transformer_blocks[0]
                mods += [tb.attn1, tb.attn2]
        tb = unet.mid_block.attentions[0].transformer_blocks[0]
        mods += [tb.attn1, tb.attn2]
        _ATTN_SITES_CACHE[unet] = mods
    return mods


def register_time(model, t):
    """Reference :20-40."""
    for module in _timed_modules(model.unet):
        module.t = t


_LATENT_CACHE = {}


def load_source_latents_t(t, latents_path):
    """Reference :43-47.  The reference re-reads the full [N,4,h,w] file on every denoise_step
    ((N/B+1) times per timestep); the tensor is kept for the current timestep instead."""
    latents_t_path = os.path.join(latents_path, f'noisy_latents_{t}.pt')
    assert os.path.exists(latents_t_path), f'Missing latents at t {t} path {latents_t_path}'
    key = (latents_t_path, os.path.getmtime(latents_t_path))
    hit = _LATENT_CACHE.get("entry")
    if hit is not None and hit[0] == key:
        return hit[1]
    latents = torch.load(latents_t_path)
    _LATENT_CACHE["entry"] = (key, latents)
    return latents


# --------------------------------------------------------------------------------------------
# injection schedules
# --------------------------------------------------------------------------------------------
def _in_schedule(module) -> bool:
    """`schedule is not None and (t in schedule or t == 1000)` (reference :86, :124) without a
    device sync: the schedule is turned into a host set once per schedule object."""
    sched = getattr(module, "injection_schedule", None)
    if sched is None:
        return False
    t = module.t
    t = int(t) if not torch.is_tensor(t) else int(t.item())
    if t == 1000:
        return True
    cached = module.__dict__.get("_tf_sched")
    if cached is None or cached[0] is not sched:
        values = sched.tolist() if torch.is_tensor(sched) else list(sched)
        cached = (sched, frozenset(int(x) for x in values))
        module.__dict__["_tf_sched"] = cached
    return t in cached[1]


def register_conv_injection(model, injection_schedule):
    """Reference :49-104: PnP feature injection in up_blocks[1].resnets[1] — the residual branch of
    the uncond and cond streams is replaced by the source stream's while t is in the schedule."""

    def make_forward(res):
        def forward(input_tensor, temb):
            skip = input_tensor
            h = norm_act(res.norm1, input_tensor)
            resample = res.upsample if res.upsample is not None else res.downsample
            if resample is not None:
                if res.upsample is not None and h.shape[0] >= 64:
                    skip, h = skip.contiguous(), h.contiguous()
                skip, h = resample(skip), resample(h)
            h = res.conv1(h)
            if temb is not None:
                temb = res.time_emb_proj(res.nonlinearity(temb))
            if res.time_embedding_norm == "default":    # temb add + norm2 + SiLU (one fused kernel on the GPU)
                h = norm_act(res.norm2, h, bias=temb)
            else:
                h = res.norm2(h)
                if temb is not None and res.time_embedding_norm == "scale_shift":
                    scale, shift = torch.chunk(temb[:, :, None, None], 2, dim=1)
                    h = h * (1 + scale) + shift
                h = res.nonlinearity(h)
            h = res.conv2(res.dropout(h))
            if _in_schedule(res):
                def inject_thirds(part):
                    n = part.shape[0] // 3
                    part[n:2 * n] = part[:n]    # uncond <- source   (:89)
                    part[2 * n:] = part[:n]     # cond   <- source   (:91)

                shard = getattr(res, "_tf_shard", None)
                n_piv = getattr(res, "_tf_fused", 0)
                if n_piv:                       # fused pass: [pivotal samples | frame samples]
                    if shard is None:
                        inject_thirds(h[:n_piv])
                    else:                       # sharded pivotal samples: the source sample may be on another rank
                        h[:n_piv] = shard.all_gather(h[:n_piv]).index_select(0, shard.source_index(h.device))
                    inject_thirds(h[n_piv:])
                else:
                    inject_thirds(h)
            if res.conv_shortcut is not None:
                skip = res.conv_shortcut(skip)
            out = skip + h
            return out if res.output_scale_factor == 1.0 else out / res.output_scale_factor
        return forward

    conv_module = model.unet.up_blocks[1].resnets[1]
    conv_module.forward = make_forward(conv_module)
    conv_module.injection_schedule = injection_schedule


# --------------------------------------------------------------------------------------------
# extended attention closures
# --------------------------------------------------------------------------------------------
_INJECTED_SITES = {1: (1, 2), 2: (0, 1, 2), 3: (0, 1, 2)}   # reference :208, :289


def _fused_weight(attn, names, dtype):
    """cat([attn.<name>.weight ...]) in `dtype`, cached on the module and re-made when any of the weights
    changes storage or version (load_state_dict, .half(), in-place updates)."""
    ws = [getattr(attn, n).weight for n in names]
    key = tuple((w.data_ptr(), w._version) for w in ws) + (dtype,)
    cache = attn.__dict__.setdefault("_tf_fused_w", {})
    hit = cache.get(names)
    if hit is None or hit[0] != key:
        hit = (key, torch.cat([w.detach().to(dtype) for w in ws], dim=0).contiguous())
        cache[names] = hit
    return hit[1]


def _row_split_attention(attn, to_out, shard, q_all, k_all, v_all, inject):
    """Extended attention of ALL 3K samples for this rank's query rows, `to_out` on those rows, all-gather, and
    re-assembly of the complete [3K, S, dim] output (stashed on the module for the block); returns the rows of the
    local samples."""
    S, dim = q_all.shape[1], q_all.shape[2]
    n_all = 3 * shard.K
    row0, nrows = shard.row_split(S)
    part = _ops().ext_attn_table(q_all, k_all, v_all, shard.global_attention_table(inject), attn.heads, attn.scale,
                                 row0=row0, nrows=nrows)                       # [3K, nrows, dim]
    if not torch.is_autocast_enabled() and part.dtype != to_out.weight.dtype:
        part = part.to(to_out.weight.dtype)
    part = to_out(part)
    full = shard.all_gather(part).view(shard.world_size, n_all, nrows, dim).permute(1, 0, 2, 3)
    full = full.reshape(n_all, shard.world_size * nrows, dim)[:, :S].contiguous()
    attn._tf_attn_full = full
    return full.index_select(0, shard.local_index(full.device))


def _sa_forward(attn, pnp: bool):
    to_out = attn.to_out[0] if type(attn.to_out) is torch.nn.modules.container.ModuleList else attn.to_out

    def fast_path(x, encoder_hidden_states):
        """fp16 activations on a GPU with fp16 GEMM operands (fp16 weights, or autocast casting them): the
        three projections run as ONE cuBLAS GEMM on the concatenated weight and q/k/v are strided views of
        its output — the kernel addresses them by token stride (SURVEY.md §8 f-3)."""
        if encoder_hidden_states is not None or not x.is_cuda or x.dtype != torch.float16:
            return False
        if any(getattr(attn, n).bias is not None for n in ("to_q", "to_k", "to_v")):
            return False
        return torch.is_autocast_enabled() or attn.to_q.weight.dtype == torch.float16

    def forward(x, encoder_hidden_states=None, attention_mask=None):
        inject = pnp and _in_schedule(attn)
        shard = getattr(attn, "_tf_shard", None)
        dim = attn.to_q.weight.shape[0]
        if fast_path(x, encoder_hidden_states):
            qkv = torch.nn.functional.linear(x, _fused_weight(attn, ("to_q", "to_k", "to_v"), torch.float16))
            q, k, v = qkv[..., :dim], qkv[..., dim:2 * dim], qkv[..., 2 * dim:]
        else:
            ctx = x if encoder_hidden_states is None else encoder_hidden_states
            q, k, v = attn.to_q(x), attn.to_k(ctx), attn.to_v(ctx)
        if shard is not None:
            # sharded pivotal pass: ONE all-gather of [q | k | v | pivot unit rows] per sample, attention of all 3K
            # samples for this rank's query rows, to_out on those rows, ONE all-gather of the result (the block picks
            # the gathered unit rows and the complete [3K, S, dim] output up from the module)
            unit = attn.__dict__.pop("_tf_unit_local", None)
            packed = shard.all_gather(torch.cat([q, k, v] + ([unit] if unit is not None else []), dim=-1))
            if unit is not None:
                # torch.cat promotes (fp16 unit rows next to fp32 q): back to the unit rows' dtype, exact
                attn._tf_unit_gathered = packed[..., 3 * dim:].to(unit.dtype)
            return _row_split_attention(attn, to_out, shard, packed[..., :dim], packed[..., dim:2 * dim],
                                        packed[..., 2 * dim:3 * dim], inject)
        out = _ops().ext_attn(q, k, v, attn.heads, attn.scale, inject)
        if not torch.is_autocast_enabled() and out.dtype != to_out.weight.dtype:
            out = out.to(to_out.weight.dtype)       # fp16 kernel output feeding a non-autocast fp32 module
        return to_out(out)

    return forward


def register_extended_attention_pnp(model, injection_schedule):
    """Reference :106-214: every block's attn1 becomes extended attention; the 8 decoder sites get
    the q/k injection schedule, all others an empty one."""
    for module in _transformer_blocks(model.unet):
        module.attn1.forward = _sa_forward(module.attn1, pnp=True)
        module.attn1.injection_schedule = []
    for res, blocks in _INJECTED_SITES.items():
        for block in blocks:
            attn1 = model.unet.up_blocks[res].attentions[block].transformer_blocks[0].attn1
            attn1.forward = _sa_forward(attn1, pnp=True)
            attn1.injection_schedule = injection_schedule


def register_extended_attention(model):
    """Reference :216-294 (SDEdit flavour: no injection)."""
    for module in _transformer_blocks(model.unet):
        module.attn1.forward = _sa_forward(module.attn1, pnp=False)


# --------------------------------------------------------------------------------------------
# TokenFlow block
# --------------------------------------------------------------------------------------------
_BLEND_CACHE = {}


def _default_frame_table(batch_idx: int, n_frames: int):
    """Reference :331-333 and :375-383 as a per-frame table."""
    from .ops import blend_weights
    w = _BLEND_CACHE.get(n_frames)
    if w is None:
        w = tuple(blend_weights(n_frames))
        _BLEND_CACHE[n_frames] = w
    kf_a = (batch_idx,) * n_frames
    kf_b = ((batch_idx - 1) if batch_idx > 0 else -1,) * n_frames
    return kf_a, kf_b, w


def make_tokenflow_attention_block(block_class: Type[torch.nn.Module]) -> Type[torch.nn.Module]:
    """Reference :296-429.  Returns a subclass of `block_class` whose forward is the TokenFlow
    block: the pivotal pass caches norm1 features and the extended-attention output of the
    keyframes; the frame pass skips attn1 and propagates keyframe rows along the NN field."""

    class TokenFlowBlock(block_class):

        def forward(self, hidden_states, attention_mask=None, encoder_hidden_states=None,
                    encoder_attention_mask=None, timestep=None, cross_attention_kwargs=None,
                    class_labels=None) -> torch.Tensor:
            if getattr(self, "use_ada_layer_norm", False) or getattr(self, "use_ada_layer_norm_zero", False):
                raise NotImplementedError(
                    "tokenflow_b200: AdaLayerNorm transformer blocks are not part of any Stable-Diffusion "
                    "UNet and are not supported by the H100 hot path")
            cross_attention_kwargs = cross_attention_kwargs if cross_attention_kwargs is not None else {}
            n_piv = getattr(self, "_tf_fused", 0)
            if n_piv:
                # fused pass: the batch is [pivotal samples | frame samples]; the keyframe caches filled by the
                # first part are consumed by the second within the same block call, so one UNet pass does the
                # work of the reference's pivotal pass + frame passes (identical arithmetic, half the launches)
                piv = self._tf_pivotal(hidden_states[:n_piv],
                                       None if encoder_hidden_states is None else encoder_hidden_states[:n_piv],
                                       cross_attention_kwargs)
                frm = self._tf_frames(hidden_states[n_piv:])
                hidden_states = torch.cat([piv, frm.to(piv.dtype) if frm.dtype != piv.dtype else frm])
            elif self.pivotal_pass:
                hidden_states = self._tf_pivotal(hidden_states, encoder_hidden_states, cross_attention_kwargs)
            else:
                hidden_states = self._tf_frames(hidden_states)

            if self.attn2 is not None:
                attn_output = self.attn2(self.norm2(hidden_states), encoder_hidden_states=encoder_hidden_states,
                                         attention_mask=encoder_attention_mask, **cross_attention_kwargs)
                hidden_states = attn_output + hidden_states
            return self.ff(self.norm3(hidden_states)) + hidden_states

        def _tf_pivotal(self, hidden_states, encoder_hidden_states, cross_attention_kwargs):
            """Self-attention stage of the pivotal pass (reference :311-327, :352-360, :394-397)."""
            ops = _ops()
            batch_size, sequence_length, dim = hidden_states.shape
            shard = getattr(self, "_tf_shard", None)
            fused_ln = (hidden_states.is_cuda and hidden_states.dtype == torch.float16
                        and hasattr(ops, "layernorm_rows") and not self.only_cross_attention
                        and (torch.is_autocast_enabled() or self.norm1.weight.dtype == torch.float16))
            # unit rows of the pivot features for the NN field: of the source stream, or, when sharded (this rank holds
            # m of the 3K (stream, keyframe) samples), of every local sample — the source samples may be on any rank
            n_unit = batch_size if shard is not None else batch_size // 3
            if fused_ln:
                # one read of hidden_states -> fp16 norm1 output (QKV operand) + its unit rows
                norm_hidden_states, unit = ops.layernorm_rows(hidden_states, self.norm1, n_unit)
            else:
                norm_hidden_states = self.norm1(hidden_states)
                unit = ops.unit_rows(norm_hidden_states[:n_unit])
            if shard is not None:
                # the unit rows ride in the attention's q|k|v all-gather, which also re-assembles the complete output
                self.attn1._tf_unit_local = unit
                self.pivot_hidden_states = norm_hidden_states
                self.attn_output = self.attn1(norm_hidden_states, **cross_attention_kwargs)
                unit_all = self.attn1.__dict__.pop("_tf_unit_gathered", None)
                full = self.attn1.__dict__.pop("_tf_attn_full", None)
                if unit_all is None or full is None:
                    raise RuntimeError("tokenflow_b200: a sharded pivotal pass needs the extended-attention attn1 of "
                                       "register_extended_attention[_pnp]; this block's attn1 did not gather the pivot "
                                       "unit rows and the attention output")
                self._tf_pivot_unit = unit_all[:shard.K].contiguous()              # source stream
                self.kf_attn_output = full
            else:
                # cache keyframe features (:326-327) — plus their fp16 unit rows for the NN field
                self._tf_pivot_unit = unit
                self.pivot_hidden_states = norm_hidden_states.view(3, n_unit, sequence_length, dim)
                self.attn_output = self.attn1(
                    norm_hidden_states,
                    encoder_hidden_states=encoder_hidden_states if self.only_cross_attention else None,
                    **cross_attention_kwargs)
                self.kf_attn_output = self.attn_output                                   # :360
            return self.attn_output + hidden_states                                      # :397

        def _tf_frames(self, hidden_states):
            """Self-attention stage of a frame pass: NN field + propagation (reference :329-348, :361-397)."""
            ops = _ops()
            batch_size, sequence_length, dim = hidden_states.shape
            n_frames = batch_size // 3
            table = getattr(self, "_tf_frame_table", None)
            if table is None:
                table = _default_frame_table(self.batch_idx, n_frames)
            kf_a, kf_b, w = table
            if len(kf_a) != n_frames:
                raise ValueError(f"frame table has {len(kf_a)} entries but the pass has {n_frames} frames")
            kf = self.kf_attn_output
            n_kf = kf.shape[0] // 3
            # norm1 of the source stream only — the other two thirds are never used in this branch (:335)
            x_unit = ops.layernorm_unit_rows(hidden_states[:n_frames], self.norm1)
            idx_a, idx_b = ops.nn_field(x_unit, self._tf_pivot_unit, kf_a, kf_b)          # :335-343
            out_dtype = torch.float32 if (_strict_dtype() and idx_b is not None) else None
            self._tf_nn_idx = (idx_a, idx_b)
            out = ops.propagate(kf.view(3, n_kf, sequence_length, dim), idx_a, idx_b, kf_a, kf_b, w,
                                residual=hidden_states, out_dtype=out_dtype)              # :361-397
            if not torch.is_autocast_enabled() and out.dtype != hidden_states.dtype and not _strict_dtype():
                out = out.to(hidden_states.dtype)    # fp16 kernel output inside a non-autocast (fp32) model
            return out

    return TokenFlowBlock


def set_tokenflow(model: torch.nn.Module):
    """Reference :432-448: swap every BasicTransformerBlock's class for the TokenFlow subclass."""
    _invalidate_cache()
    made = {}
    for _, module in model.named_modules():
        if isinstance_str(module, "BasicTransformerBlock") and not isinstance_str(module, "TokenFlowBlock"):
            cls = module.__class__
            if cls not in made:
                made[cls] = make_tokenflow_attention_block(cls)
            module.__class__ = made[cls]
            if not hasattr(module, "use_ada_layer_norm_zero"):
                module.use_ada_layer_norm = False
                module.use_ada_layer_norm_zero = False
    return model
