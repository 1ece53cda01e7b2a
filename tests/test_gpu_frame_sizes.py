"""GPU tier of frame resizing and non-square latents.

* `tf_resize_u8` equals PIL's LANCZOS resize byte for byte at the frame sizes users bring (1080p and 720p landscape,
  portrait, square, upscaling, one axis only), for one frame and for 40, and writes exactly its output: `tmp` and `out`
  sit between sentinel-filled guard bands, and the intermediate equals PIL's horizontal-only resize.
* The hot-path kernels at the token counts of non-square videos: SD1.5 at 384 x 672 (S = 4032, 1008, 252, 66) and
  360 x 640 (S = 3600, 920, 240, 60), SD2.1 at 384 x 672, at production head counts.  S = 66 and 60 are below one key
  tile, the others are not tile multiples, and a multi-GPU row split leaves trailing ranks without rows.
* The hook layer, the CUDA-graphed editor step and the whole frames-to-frames chain at 48 x 84 latents.
"""
import numpy as np
import pytest
import torch
from PIL import Image

from oracle import tokenflow_oracle as O
from oracle.kernel_checks import check_ext_attn, check_group_norm, check_nn_field, ext_attn_samples
from oracle.kernel_checks import tie_class as tie_class_of
from oracle.oracle_ops import OracleOps
from tokenflow_b200 import ops as ops_module
from tokenflow_b200 import sd_unet
from tokenflow_b200 import tokenflow_utils as tfu
from tokenflow_b200.editor import TokenFlowEditor, synthetic_inputs
from tokenflow_b200.ops import blend_weights
from tokenflow_b200.scheduler import DDIMScheduler

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5


@pytest.fixture(scope="module")
def ops():
    from tokenflow_b200.ops import CudaOps
    return CudaOps()


def _content(kind, n, h, w, seed):
    rng = np.random.default_rng(seed)
    if kind == "random":
        return rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8)
    yy, xx = np.mgrid[0:h, 0:w]
    if kind == "checker":               # 0 / 255 cells of a few sizes: Lanczos rings at every edge, both clamps bite
        base = np.stack([((yy // (1 + f) + xx // (2 + f)) % 2) * 255 for f in range(3)], -1).astype(np.uint8)
    else:                               # hard edges plus a ramp
        base = np.stack([(xx >= w // 3) * 255, (yy >= h // 2) * 255, (xx * 255) // max(w - 1, 1)], -1).astype(np.uint8)
    frames = np.repeat(base[None], n, axis=0)
    frames[1::2] = 255 - frames[1::2]
    return frames


def _pil(frames, h, w):
    return np.stack([np.asarray(Image.fromarray(f).resize((w, h), Image.LANCZOS)) for f in frames])


def _guarded(numel, guard):
    buf = torch.full((guard + numel + guard,), SENTINEL, dtype=torch.uint8, device="cuda")
    return buf, buf[guard:guard + numel]


CASES = [  # (H_in, W_in) -> (H, W)
    ((1080, 1920), (384, 672)),
    ((1080, 1920), (360, 640)),
    ((1080, 1080), (512, 512)),
    ((1280, 720), (672, 384)),
    ((240, 320), (384, 672)),          # upscaling
    ((720, 1280), (720, 672)),         # horizontal only
    ((720, 1280), (384, 1280)),        # vertical only
    ((97, 131), (53, 29)),             # odd sizes: byte-wise vertical path, unaligned rows
]


@pytest.mark.parametrize("n", [1, 40])
@pytest.mark.parametrize("kind", ["random", "checker", "edges"])
@pytest.mark.parametrize("src,dst", CASES, ids=[f"{a[1]}x{a[0]}-{b[1]}x{b[0]}" for a, b in CASES])
def test_resize_equals_pil(ops, src, dst, kind, n):
    if n == 40 and kind != "random" and src[0] * src[1] > 1280 * 720:
        pytest.skip("40 frames of 1080p once per size, with random content")
    (h_in, w_in), (h, w) = src, dst
    frames = _content(kind, n, h_in, w_in, seed=h_in + w + n)
    want = _pil(frames, h, w)
    guard = 256 + (h_in + w) % 7                                # odd guards: unaligned tmp / out as well
    tbuf, tmp = _guarded(n * h_in * w * 3, guard)
    obuf, out = _guarded(n * h * w * 3, guard + 3)
    got = ops.resize_frames(torch.from_numpy(frames).cuda(), (h, w), tmp=tmp.view(n, h_in, w, 3),
                            out=out.view(n, h, w, 3))
    torch.cuda.synchronize()
    assert got.data_ptr() == out.data_ptr()
    bad = (got.cpu().numpy() != want)
    assert not bad.any(), f"{int(bad.sum())} of {bad.size} bytes differ from PIL"
    for buf, g in ((tbuf, guard), (obuf, guard + 3)):
        assert bool((buf[:g] == SENTINEL).all()) and bool((buf[buf.numel() - g:] == SENTINEL).all())
    if w != w_in and h != h_in:              # both passes: the intermediate is PIL's horizontal-only resize
        assert np.array_equal(tmp.view(n, h_in, w, 3).cpu().numpy(), _pil(frames, h_in, w))
    else:                                    # one pass or none: tmp is not touched
        assert bool((tbuf == SENTINEL).all())


def test_resize_identity_is_a_copy_and_launches_nothing(ops):
    frames = torch.from_numpy(_content("random", 3, 64, 96, 1)).cuda()
    before = ops.launch_count()
    got = ops.resize_frames(frames, (64, 96))
    assert ops.launch_count() == before and got.data_ptr() != frames.data_ptr() and torch.equal(got, frames)
    two = ops.resize_frames(frames, (32, 48))
    assert ops.launch_count() - before == 2 and two.shape == (3, 32, 48, 3)


def test_preprocess_resize_frames_device_equals_host():
    from tokenflow_b200.preprocess import resize_frames
    frames = torch.from_numpy(_content("random", 4, 720, 1280, 3))
    assert torch.equal(resize_frames(frames.cuda(), (384, 672)).cpu(), resize_frames(frames, (384, 672)))
    sq = torch.from_numpy(_content("edges", 2, 720, 720, 4))
    assert torch.equal(resize_frames(sq.cuda(), 512).cpu(), resize_frames(sq, 512))


# ------------------------------------------------------------------------------------------------
# the kernels at the token counts of non-square videos
# ------------------------------------------------------------------------------------------------
def _levels(latent_hw):
    h, w = latent_hw
    out = []
    for _ in range(4):
        out.append(h * w)
        h, w = (h + 1) // 2, (w + 1) // 2
    return out


SD15_DIMS, SD15_HEADS = (320, 640, 1280, 1280), (8, 8, 8, 8)
SD21_HEADS = (5, 10, 20, 20)
KERNEL_CASES = []
for name, lat, heads in (("sd15-384x672", (48, 84), SD15_HEADS), ("sd15-360x640", (45, 80), SD15_HEADS),
                         ("sd21-384x672", (48, 84), SD21_HEADS)):
    for lvl, S in enumerate(_levels(lat)):
        KERNEL_CASES.append(pytest.param(S, SD15_DIMS[lvl], heads[lvl], id=f"{name}-S{S}"))


@pytest.mark.parametrize("S,dim,heads", KERNEL_CASES)
@pytest.mark.parametrize("inject", [False, True])
def test_ext_attn_at_non_square_token_counts(ops, S, dim, heads, inject):
    torch.manual_seed(S + dim)
    n, d = 3, dim // heads
    q = torch.randn(3 * n, S, dim, device="cuda")
    k = (torch.randn(3 * n, S, dim, device="cuda") + q).half()               # peaked rows, as in video features
    q, v = q.half(), torch.randn(3 * n, S, dim, device="cuda").half()
    table = ext_attn_samples(n, inject)
    whole = ops.ext_attn(q, k, v, heads, d ** -0.5, inject)
    check_ext_attn(whole, q, k, v, table, heads, d ** -0.5, atol=2.5e-3, max_rel=1e-3)
    for G in (2, 8):                        # the multi-GPU query-row split, trailing ranks past S included
        parts = []
        for r in range(G):
            row0, nrows = tfu.PivotalShard(G, r, n).row_split(S)
            parts.append(ops.ext_attn_table(q, k, v, table, heads, d ** -0.5, row0=row0, nrows=nrows))
        nrows = parts[0].shape[1]
        got = torch.stack(parts).permute(1, 0, 2, 3).reshape(3 * n, G * nrows, dim)[:, :S]
        if nrows >= 256 or S <= 128:
            assert torch.equal(got, whole), (G, (got.float() - whole.float()).abs().max().item())
        else:                               # one-tile ranges run the one-tile kernel: same math, other tiling
            check_ext_attn(got, q, k, v, table, heads, d ** -0.5, atol=2.5e-3, max_rel=1e-3)


@pytest.mark.parametrize("S,dim,heads", KERNEL_CASES)
def test_nn_field_and_propagate_at_non_square_token_counts(ops, S, dim, heads):
    torch.manual_seed(S * 3 + dim)
    K, B = 5, 8
    F = 2 * B
    piv = torch.nn.functional.layer_norm(torch.randn(K, S, dim, device="cuda"), (dim,))
    kf_a = [1 + f // B for f in range(F)]
    kf_b = [a - 1 for a in kf_a]
    x = torch.stack([piv[a][torch.randperm(S, device="cuda")] for a in kf_a]) + 0.3 * torch.randn(F, S, dim, device="cuda")
    xu, pu = ops.unit_rows(x), ops.unit_rows(piv)
    idx_a, idx_b = ops.nn_field(xu, pu, kf_a, kf_b)
    check_nn_field(idx_a, idx_b, xu, pu, kf_a, kf_b)
    w = [blend_weights(B)[f % B] for f in range(F)]
    A = torch.randn(3, K, S, dim, device="cuda").half()
    res = torch.randn(3 * F, S, dim, device="cuda").half()
    got = ops.propagate(A, idx_a, idx_b, kf_a, kf_b, w, res)
    want = OracleOps().propagate(A, idx_a, idx_b, kf_a, kf_b, w, res).half()
    assert torch.equal(got, want)


@pytest.mark.parametrize("kind", ["sd15", "sd21"])
def test_every_group_norm_site_at_48x84(kind, monkeypatch):
    body = ops_module.body_ops()
    assert body is not None
    unet = sd_unet.build_unet(kind, seed=1, device="cuda", dtype=torch.float16, init_on_device=True)
    unet = unet.to(memory_format=torch.channels_last)
    g = torch.Generator(device="cuda").manual_seed(0)
    sample = torch.randn(2, 4, 48, 84, device="cuda", generator=g).half().contiguous(memory_format=torch.channels_last)
    ctx = torch.randn(2, 77, unet.config.cross_attention_dim, device="cuda", generator=g).half()
    calls = []
    native = body.group_norm_nhwc

    def record(x, norm, bias=None, silu=False):
        out = native(x, norm, bias, silu)
        calls.append((x.clone(), norm, None if bias is None else bias.clone(), silu, out.clone()))
        return out

    monkeypatch.setattr(body, "group_norm_nhwc", record)
    with torch.no_grad():
        out = unet(sample, torch.tensor([501], device="cuda"), encoder_hidden_states=ctx).sample
    monkeypatch.undo()
    assert out.shape == (2, 4, 48, 84) and torch.isfinite(out).all()
    assert len(calls) == 61
    sizes = set()
    for i, (x, norm, bias, silu, y) in enumerate(calls):
        sizes.add(tuple(x.shape[-2:]))
        check_group_norm(y, x, norm, bias, silu, f"{kind} 48x84 site {i} {tuple(x.shape)}", exempt_aten_misrounded=True)
    assert sizes == {(48, 84), (24, 42), (12, 21), (6, 11)}


# ------------------------------------------------------------------------------------------------
# hooks, editor and the frames-to-frames chain at 48 x 84 latents
# ------------------------------------------------------------------------------------------------
def _run_tiny(ops_obj, mode, steps, latent=(48, 84), n_frames=4, batch=2, seed=1):
    tfu._install_ops_for_testing(ops_obj)
    unet = sd_unet.build_unet("tiny", seed=seed, device="cuda", dtype=torch.float16)
    cfg = {"n_frames": n_frames, "batch_size": batch, "n_timesteps": steps, "guidance_scale": 7.5,
           "mode": mode, "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "start": 0.9}
    x, text, pnp, src = synthetic_inputs(n_frames, latent, unet.config.cross_attention_dim, steps, seed=seed,
                                         device="cuda", dtype=torch.float16, ctx_len=7)
    ed = TokenFlowEditor(unet, DDIMScheduler(), tfu, cfg, text, pnp, source_latents=lambda t: src[t])
    ed.init_method()
    torch.manual_seed(seed)
    return ed.sample_loop(x).float(), ed.keyframe_log


@pytest.mark.parametrize("mode,steps", [("pnp", 2), ("sdedit", 10)])
def test_tiny_unet_edit_at_48x84_cuda_vs_reference_gpu_path(mode, steps):
    want, kf_w = _run_tiny(OracleOps(), mode, steps)
    got, kf_g = _run_tiny(None, mode, steps)
    assert kf_g == kf_w and got.shape == (4, 4, 48, 84) and torch.isfinite(got).all()
    rel = (got - want).norm() / want.norm()
    assert rel.item() < 2e-2, rel.item()


class _U(torch.nn.Module):
    def __init__(self, block):
        super().__init__()
        site = torch.nn.Module()
        site.transformer_blocks = torch.nn.ModuleList([block])
        ups = []
        for _ in range(4):
            u = torch.nn.Module()
            u.attentions = torch.nn.ModuleList([site, site, site])
            ups.append(u)
        self.up_blocks = torch.nn.ModuleList(ups)


class _W(torch.nn.Module):
    def __init__(self, unet):
        super().__init__()
        self.unet = unet


@pytest.mark.parametrize("inject", [False, True])
def test_sd15_block_at_4032_tokens_vs_reference_gpu_path(inject):
    """The SD1.5 top-level block of a 384 x 672 video (S = 4032, dim 320, 8 heads x 40), K = 5, B = 8, PnP flavour:
    pivotal pass + frame passes 0 and 2, CUDA ops vs oracle ops under the same autocast.  Every NN-index mismatch lies
    inside an fp16 tie class of the oracle's own similarity values."""
    K, B, S, dim = 5, 8, 4032, 320

    def run(ops_obj):
        tfu._install_ops_for_testing(ops_obj)
        torch.manual_seed(3)
        block = sd_unet.BasicTransformerBlock(dim, 8, 40, 768).cuda().half().eval()
        model = _W(_U(block))
        sched = [981, 961]
        tfu.register_extended_attention_pnp(model, sched)
        block.attn1.injection_schedule = sched
        tfu.set_tokenflow(model.unet)
        block.attn1.t = 981 if inject else 1
        res = {}
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
            h = torch.randn(3 * K, S, dim, device="cuda").half()
            ctx = torch.randn(3 * K, 77, 768, device="cuda").half()
            tfu.register_pivotal(model, True)
            res["piv"] = block(h, encoder_hidden_states=ctx).float()
            tfu.register_pivotal(model, False)
            for i in (0, 2):
                hf = h[:K][i].unsqueeze(0).repeat(B, 1, 1) + 0.3 * torch.randn(B, S, dim, device="cuda").half()
                hf = torch.cat([hf, torch.randn(2 * B, S, dim, device="cuda").half()])
                tfu.register_batch_idx(model, i)
                res[f"out{i}"] = block(hf, encoder_hidden_states=torch.randn(3 * B, 77, 768, device="cuda").half()).float()
                res[f"idx{i}"] = tuple(None if t is None else t.long().reshape(B, S).clone() for t in block._tf_nn_idx)
                res[f"x{i}"] = hf[:B].clone()
        res["block"] = block
        return res

    want, got = run(OracleOps()), run(None)
    assert torch.allclose(got["piv"], want["piv"], atol=4e-3, rtol=4e-3)
    total = mismatched = ties = 0
    for i in (0, 2):
        same = torch.ones((B, S), dtype=torch.bool, device="cuda")
        for which in (0, 1):
            g_idx, w_idx = got[f"idx{i}"][which], want[f"idx{i}"][which]
            if g_idx is None:
                assert w_idx is None
                continue
            bad = g_idx != w_idx
            same &= ~bad
            total += g_idx.numel()
            mismatched += int(bad.sum())
            if bad.any():
                blk = want["block"]
                with torch.autocast("cuda", dtype=torch.float16):
                    sim = O.cosine_sim(blk.norm1(want[f"x{i}"]).reshape(-1, dim),
                                       blk.pivot_hidden_states[0][i if which == 0 else i - 1])
                rows = bad.reshape(-1).nonzero().squeeze(1)
                ties += int(tie_class_of(sim, rows, g_idx.reshape(-1)[rows], w_idx.reshape(-1)[rows], ulps=2).sum())
        rows = same.reshape(1, -1).expand(3, -1).reshape(-1)
        assert torch.allclose(got[f"out{i}"].reshape(-1, dim)[rows], want[f"out{i}"].reshape(-1, dim)[rows],
                              atol=4e-3, rtol=4e-3)
    msg = f"NN indices: {mismatched} of {total} differ, {ties} of them inside an fp16 tie class"
    print(msg)
    assert mismatched == ties and mismatched <= 5e-3 * total, msg


def test_cuda_graph_step_identical_to_eager_at_48x84():
    """SD1.5, 8 frames, B = 4, 5 PnP steps at 48 x 84 latents: the three captured step variants (q/k + conv injection,
    conv injection only, none) replay to the eager step's bits."""
    def editor(graph):
        tfu._install_ops_for_testing(None)
        unet = sd_unet.build_unet("sd15", seed=1, device="cuda", dtype=torch.float16, init_on_device=True)
        unet = unet.to(memory_format=torch.channels_last)
        cfg = {"n_frames": 8, "batch_size": 4, "n_timesteps": 5, "guidance_scale": 7.5, "mode": "pnp",
               "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "fused_pass": True, "cuda_graph": graph, "keyframe_seed": 1}
        x, text, pnp, src = synthetic_inputs(8, (48, 84), unet.config.cross_attention_dim, 5, seed=1, device="cuda",
                                             dtype=torch.float16, ctx_len=7)
        ed = TokenFlowEditor(unet, DDIMScheduler(), tfu, cfg, text, pnp, source_latents=lambda t: src[t])
        ed.init_method()
        return ed, x

    ed_e, x = editor(False)
    want = ed_e.sample_loop(x.clone())
    del ed_e
    ed_g, x = editor(True)
    got = ed_g.sample_loop(x.clone())
    assert len(ed_g._graphs) == 3 and all(e["replays"] >= 1 for e in ed_g._graphs.values())
    assert got.shape == (8, 4, 48, 84) and torch.isfinite(got).all()
    assert torch.equal(got, want), (got.float() - want.float()).abs().max().item()


@torch.no_grad()
def test_native_size_frames_to_edited_frames():
    """1280 x 720 uint8 frames -> resize_frames on the device -> encode -> 4 inversion steps -> 4 PnP steps -> decode ->
    672 x 384 uint8 frames, equal to the same chain fed by PIL's resize on the host (SD VAE, tiny UNet)."""
    from tokenflow_b200.preprocess import LatentInverter, ddim_eps, decode_latents, encode_imgs, resize_frames
    from tokenflow_b200.vae import build_vae
    tfu._install_ops_for_testing(None)
    vae = build_vae("sd", seed=1, device="cuda", dtype=torch.float16,
                    init_on_device=True).to(memory_format=torch.channels_last)
    n, steps = 4, 4
    g = torch.Generator().manual_seed(5)
    low = torch.rand(n, 3, 9, 16, generator=g)
    img = torch.nn.functional.interpolate(low, size=(720, 1280), mode="bicubic", align_corners=False)
    frames = ((img + 0.05 * torch.randn(n, 3, 720, 1280, generator=g)).clamp(0, 1) * 255).round().to(torch.uint8)
    frames = frames.permute(0, 2, 3, 1).contiguous()
    unet_kw = dict(seed=1, device="cuda", dtype=torch.float16)
    ctx = sd_unet.tiny_config().cross_attention_dim
    pnp = torch.randn(1, 7, ctx, generator=g).half().cuda()
    text = torch.randn(2, 7, ctx, generator=g).half().cuda()
    cfg = {"n_frames": n, "batch_size": 2, "n_timesteps": steps, "guidance_scale": 7.5, "mode": "pnp",
           "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "fused_pass": True, "cuda_graph": True, "keyframe_seed": 1}

    def chain(resized):
        latents = encode_imgs(vae, resized, batch_size=2)
        assert latents.shape == (n, 4, 48, 84)
        unet = sd_unet.build_unet("tiny", **unet_kw).to(memory_format=torch.channels_last)
        inv = LatentInverter(unet, DDIMScheduler(), steps)
        inv.ddim_inversion(pnp, latents, None, batch_size=2, save_latents=False)
        saved = inv.saved_latents()
        ed = TokenFlowEditor(sd_unet.build_unet("tiny", **unet_kw).to(memory_format=torch.channels_last),
                             DDIMScheduler(), tfu, cfg, text, pnp, source_latents=saved.__getitem__)
        x = ed.scheduler.add_noise(latents, ddim_eps(latents, saved, ed.scheduler), ed.scheduler.timesteps[0])
        ed.init_method()
        out = ed.sample_loop(x)
        assert torch.isfinite(out).all()
        return decode_latents(vae, out, batch_size=2)

    on_device = resize_frames(frames.cuda(), (384, 672))
    on_host = resize_frames(frames, (384, 672))
    assert torch.equal(on_device.cpu(), on_host)
    got = chain(on_device)
    want = chain(on_host.cuda())
    assert got.dtype == torch.uint8 and got.shape == (n, 384, 672, 3)
    assert torch.equal(got, want)
