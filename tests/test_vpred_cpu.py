"""CPU tier: v-prediction (Stable Diffusion 2.x at 768^2) through the scheduler, the inversion loop, the C ABI and the
editor.

* Ideal denoiser.  A model that knows the clean latents returns the exact eps, or the exact v, of any latent it is
  given.  Through `DDIMScheduler.step` the eps model and the v model keep every latent on the trajectory
  sqrt(a_prev) x0 + sqrt(1 - a_prev) eps0; through `LatentInverter`'s eager loop (inversion, then reconstruction) the
  two models agree.  A wrong sign, swapped coefficients or the eps formula applied to v break both.
* Planted variants.  A restatement of tf_cfg_ddim_v with one deliberate change each must differ from
  oracle/latent_step_v.py's `cfg_ddim_v` on the GPU sweep's inputs; unchanged, it must agree.
* `DDIMScheduler.from_config` on the shapes of the SD 1.5, SD 2.1-base and SD 2.1 (768-v) scheduler configs, and its
  refusals.
* A tiny-UNet v edit: the fused step equals the reference's per-batch schedule, and two gloo ranks equal one.
"""
import functools
import os
import re
import tempfile
import types

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import latent_step as LS
from oracle import latent_step_v as LSV
from tokenflow_b200 import tokenflow_utils as tfu
from tokenflow_b200.editor import TokenFlowEditor
from tokenflow_b200.preprocess import LatentInverter, inversion_coef_tables
from tokenflow_b200.scheduler import DDIMScheduler

V = "v_prediction"


# ------------------------------------------------------------------------------------------------
# a. ideal-denoiser semantics
# ------------------------------------------------------------------------------------------------
class _Ideal(torch.nn.Module):
    """Knows the clean latents x0; for a latent x at level a (looked up from the timestep it is called with) returns
    the exact eps = (x - sqrt(a) x0) / sqrt(1 - a), or v = sqrt(a) eps - sqrt(1 - a) x0, in fp64."""

    def __init__(self, x0, kind, level):
        super().__init__()
        self.p = torch.nn.Parameter(torch.zeros((), dtype=x0.dtype))
        self.x0, self.kind, self.level = x0.double(), kind, level

    def forward(self, x, t, encoder_hidden_states=None):
        a = self.level[int(t)]
        eps = (x.double() - a ** 0.5 * self.x0) / (1 - a) ** 0.5
        out = eps if self.kind == "epsilon" else a ** 0.5 * eps - (1 - a) ** 0.5 * self.x0
        return {"sample": out.to(x.dtype)}


def _latents(seed=0, shape=(3, 4, 6, 5)):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g, dtype=torch.float64), torch.randn(shape, generator=g, dtype=torch.float64)


@pytest.mark.parametrize("kind", ["epsilon", V])
def test_ideal_denoiser_stays_on_the_trajectory_through_the_step(kind):
    x0, eps0 = _latents()
    sch = DDIMScheduler(prediction_type=kind)
    sch.set_timesteps(50)
    level = {int(t): float(sch._alpha(int(t))) for t in sch.timesteps}
    model = _Ideal(x0, kind, level)
    a_T = level[int(sch.timesteps[0])]
    x = a_T ** 0.5 * x0 + (1 - a_T) ** 0.5 * eps0
    for t in sch.timesteps:
        x = sch.step(model(x, t)["sample"], t, x)["prev_sample"]
        a_prev = float(sch._alpha(int(t) - 1000 // 50))
        want = a_prev ** 0.5 * x0 + (1 - a_prev) ** 0.5 * eps0
        assert (x - want).abs().max().item() < 1e-12, int(t)


def test_the_eps_step_applied_to_v_leaves_the_trajectory():
    x0, eps0 = _latents()
    sch = DDIMScheduler()
    sch.set_timesteps(50)
    level = {int(t): float(sch._alpha(int(t))) for t in sch.timesteps}
    t = sch.timesteps[10]
    a = level[int(t)]
    x = a ** 0.5 * x0 + (1 - a) ** 0.5 * eps0
    x_prev = sch.step(_Ideal(x0, V, level)(x, t)["sample"], t, x)["prev_sample"]
    a_prev = float(sch._alpha(int(t) - 20))
    assert (x_prev - (a_prev ** 0.5 * x0 + (1 - a_prev) ** 0.5 * eps0)).abs().max().item() > 0.1


INV_STEPS = 10


def _invert_and_reconstruct(kind, x0):
    """LatentInverter's eager loop on fp32 latents (inversion, then reconstruction) with the ideal model.  The model
    is told the level at which the loop treats its input: an inversion step at t updates a sample at the level of
    the previous (less noisy) timestep; a reconstruction step at t one at the level of t."""
    sch = DDIMScheduler(prediction_type=kind)
    inv = LatentInverter(_Ideal(x0, kind, {}), sch, INV_STEPS)
    ts_up = [int(t) for t in reversed(sch.timesteps.tolist())]
    a = lambda t: float(sch.alphas_cumprod[t]) if t is not None else float(sch.final_alpha_cumprod)
    inv.unet.level = {t: a(ts_up[i - 1] if i else None) for i, t in enumerate(ts_up)}
    cond = torch.zeros(1, 7, 16)
    xT = inv.ddim_inversion(cond, x0.float(), None, batch_size=x0.shape[0], save_latents=False)
    inv.unet.level = {t: a(t) for t in ts_up}
    rec = inv.ddim_sample(xT.clone(), cond, batch_size=x0.shape[0])
    return xT.double(), rec.double(), sch, ts_up


def test_ideal_denoiser_eps_and_v_agree_through_the_eager_inversion_loop():
    x0, _ = _latents(1)
    xT_e, rec_e, sch, ts_up = _invert_and_reconstruct("epsilon", x0)
    xT_v, rec_v, _, _ = _invert_and_reconstruct(V, x0)
    # Exact arithmetic: the model's x0 is the clean latent and every step keeps x = sqrt(a) x0 + sqrt(1 - a) E for one
    # fixed E = (x0 - sqrt(a_f) x0) / sqrt(1 - a_f) (a_f = final_alpha_cumprod, the level the loop gives x0), so
    # x_T = sqrt(a_T) x0 + sqrt(1 - a_T) E and the reconstruction returns x0.  In fp32 every coefficient and every
    # operation is rounded to 2^-24 relative; an error of x is scaled by at most sqrt(1 - a') / sqrt(1 - a) <=
    # 1 / sqrt(1 - a_f) by the remaining steps, so |error| <= 2 * 12 * steps * 2^-24 * max|x| / sqrt(1 - a_f)
    # (12 rounded operations per step and direction, both directions).
    a_f, a_T = float(sch.final_alpha_cumprod), float(sch.alphas_cumprod[ts_up[-1]])
    E = (x0 - a_f ** 0.5 * x0) / (1 - a_f) ** 0.5
    scale = max(x0.abs().max().item(), E.abs().max().item())
    tol = 2 * 12 * INV_STEPS * 2.0 ** -24 * scale / (1 - a_f) ** 0.5
    want_T = a_T ** 0.5 * x0 + (1 - a_T) ** 0.5 * E
    for name, got, want in (("eps xT", xT_e, want_T), ("v xT", xT_v, want_T), ("eps rec", rec_e, x0),
                            ("v rec", rec_v, x0)):
        assert (got - want).abs().max().item() < tol, (name, (got - want).abs().max().item(), tol)
    assert (xT_e - xT_v).abs().max().item() < tol and (rec_e - rec_v).abs().max().item() < tol


def test_v_coefficient_tables_follow_the_v_branch():
    """tf_ddim_v's rows are the 0-dim fp32 alphas of the eps rows: (mu_prev, sigma_prev, mu, sigma) and (mu, sigma,
    mu_prev, sigma_prev); an eps scheduler's tables are unchanged."""
    eps, v = DDIMScheduler(), DDIMScheduler(prediction_type=V)
    for s in (eps, v):
        s.set_timesteps(500)
    (inv_e, rec_e), (inv_v, rec_v) = inversion_coef_tables(eps), inversion_coef_tables(v)
    assert torch.equal(inv_v[:, 2:], inv_e[:, 2:]) and torch.equal(inv_v[:, 1], inv_e[:, 0])
    a = eps.alphas_cumprod
    ts_up = [int(t) for t in reversed(eps.timesteps.tolist())]
    assert torch.equal(inv_v[1, 0], a[ts_up[0]] ** 0.5) and torch.equal(inv_v[0, 0], eps.final_alpha_cumprod ** 0.5)
    assert torch.equal(rec_v[:, 2:], rec_e[:, 2:]) and torch.equal(rec_v[:, 1], rec_e[:, 0])
    assert torch.equal(rec_v[:, 0], torch.stack([a[t] ** 0.5 for t in ts_up[::-1]]))


# ------------------------------------------------------------------------------------------------
# b. planted variants of tf_cfg_ddim_v
# ------------------------------------------------------------------------------------------------
STEPS = 50
GUIDANCE = 7.5


def _schedule(kind=V):
    sch = DDIMScheduler(prediction_type=kind)
    sch.set_timesteps(STEPS)
    return sch


@functools.lru_cache(maxsize=None)
def _coef_rows(kind=V):
    sch = _schedule(kind)
    stub = types.SimpleNamespace(scheduler=sch, _t_host=[int(t) for t in sch.timesteps], device="cpu")
    return TokenFlowEditor._make_coef_table(stub).numpy()


def _fp64_coefs(row):
    sch = _schedule()
    t = int(sch.timesteps[row])
    a_t, a_prev = float(sch._alpha(t)), float(sch._alpha(t - 1000 // STEPS))
    return a_t ** 0.5, (1 - a_t) ** 0.5, a_prev ** 0.5, (1 - a_prev) ** 0.5


def _cfg_ddim_v(u, c, x, row, g, *, swap_ab=False, flip_bv=False, eps_by_division=False, fma_sum=False,
                raw_ax=False, fp64=False, eps_sequence=False):
    """tf_cfg_ddim_v's arithmetic written out again; each keyword is one plausible kernel or host bug."""
    h = lambda v: v.astype(np.float16).astype(np.float32)
    u, c, x = (v.astype(np.float32) for v in (u, c, x))
    a, b, cc, d = (np.float32(k) for k in _coef_rows()[row])
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        v = h(u + h(np.float32(g) * h(c - u)))
        if eps_sequence:        # the eps kernel on v, with the eps schedule's row
            return LS.ddim_half(v, x, _coef_rows("epsilon")[row]).astype(np.float16)
        if fp64:
            hd = lambda z: z.astype(np.float16).astype(np.float64)
            A, B, C, D = _fp64_coefs(row)
            v64, x64 = v.astype(np.float64), x.astype(np.float64)
            p = hd(hd(A * x64) - hd(B * v64))
            e = hd(hd(A * v64) + hd(B * x64))
            return hd(hd(C * p) + hd(D * e)).astype(np.float16)
        if swap_ab:
            a, b = b, a
        ax = (a * x) if raw_ax else h(a * x)
        p = h(ax + h(b * v)) if flip_bv else h(ax - h(b * v))
        e = h(h(x - h(a * p)) / b) if eps_by_division else h(h(a * v) + h(b * x))
        cp, de = h(cc * p), h(d * e)
        if fma_sum:             # c * p + h(d * e) contracted: one rounding of the exact product-sum
            return (cc.astype(np.float64) * p.astype(np.float64) + de).astype(np.float32).astype(np.float16)
        return h(cp + de).astype(np.float16)


def _sweep_chunks(step=1):
    s = LS.structured_fp16()
    u = np.broadcast_to(LS.ALL_FP16[None, :], (len(s), 1 << 16))
    c = np.broadcast_to(s[:, None], u.shape)
    for xv in s[::step]:
        yield u, c, np.full(u.shape, xv, dtype=np.float16)


def _differs(row, g, step=1, **variant):
    coef = _coef_rows()[row]
    for u, c, x in _sweep_chunks(step):
        if not LS.same_bits(_cfg_ddim_v(u, c, x, row, g, **variant), LSV.cfg_ddim_v(u, c, x, coef, g)).all():
            return True
    return False


def test_restatement_on_hand_computed_values():
    f16 = lambda *v: np.array(v, np.float16)
    # a = 1, b = 0: pred_x0 = x, pred_eps = v; out = c x + d v
    assert LSV.ddim_v(f16(2), f16(3), (1.0, 0.0, 0.5, 0.25))[0] == 2.0
    # a = 0, b = 1: pred_x0 = -v, pred_eps = x
    assert LSV.ddim_v(f16(1), f16(4), (0.0, 1.0, 1.0, 1.0))[0] == 3.0
    # guidance first: v = u + g (c - u) = 1 + 2 * 1 = 3, then a = 1, b = 0, c = 1, d = 1: out = x + v
    assert LSV.cfg_ddim_v(f16(1), f16(2), f16(0.5), (1.0, 0.0, 1.0, 1.0), 2.0)[0] == 3.5
    # inf - inf in pred_x0 is NaN
    assert np.isnan(LSV.ddim_v(f16(np.inf), f16(np.inf), (1.0, 1.0, 1.0, 0.0))[0])


@pytest.mark.parametrize("row,g", [(0, GUIDANCE), (21, 3.3), (49, 0.0)])
def test_unchanged_restatement_agrees_with_the_oracle(row, g):
    assert not _differs(row, g, step=7)


# variant -> the schedule step at which it must be told apart.  fp64 coefficients change the fp16 outputs only at some
# steps (the first is 20 of 50): elsewhere no fp32 rounding of a coefficient moves a product across an fp16 boundary.
VARIANTS = {
    "a_b_swapped": (dict(swap_ab=True), 0),
    "sign_of_b_v_flipped": (dict(flip_bv=True), 0),
    "eps_from_x0_by_division": (dict(eps_by_division=True), 0),
    "fma_contracted_final_sum": (dict(fma_sum=True), 0),
    "unrounded_a_times_x": (dict(raw_ax=True), 0),
    "fp64_coefficients": (dict(fp64=True), 20),
    "eps_kernel_sequence_on_v": (dict(eps_sequence=True), 0),
}


@pytest.mark.parametrize("name", sorted(VARIANTS))
def test_sweep_tells_the_planted_variant_apart(name):
    variant, row = VARIANTS[name]
    assert _differs(row, GUIDANCE, **variant), f"{name} is indistinguishable at step {row}"


# ------------------------------------------------------------------------------------------------
# c. DDIMScheduler.from_config
# ------------------------------------------------------------------------------------------------
SD15 = {"_class_name": "PNDMScheduler", "_diffusers_version": "0.6.0", "beta_end": 0.012,
        "beta_schedule": "scaled_linear", "beta_start": 0.00085, "num_train_timesteps": 1000, "set_alpha_to_one": False,
        "skip_prk_steps": True, "steps_offset": 1, "trained_betas": None, "clip_sample": False}
SD21_BASE = {"_class_name": "DDIMScheduler", "_diffusers_version": "0.8.0", "beta_end": 0.012,
             "beta_schedule": "scaled_linear", "beta_start": 0.00085, "clip_sample": False, "num_train_timesteps": 1000,
             "prediction_type": "epsilon", "set_alpha_to_one": False, "skip_prk_steps": True, "steps_offset": 1,
             "trained_betas": None}
SD21_V = dict(SD21_BASE, prediction_type="v_prediction")


@pytest.mark.parametrize("config,kind", [(SD15, "epsilon"), (SD21_BASE, "epsilon"), (SD21_V, V)],
                         ids=["sd15", "sd21-base", "sd21-768-v"])
def test_from_config_reads_real_checkpoint_configs(config, kind):
    sch = DDIMScheduler.from_config(config)
    assert sch.prediction_type == kind
    ref = DDIMScheduler()
    assert torch.equal(sch.alphas_cumprod, ref.alphas_cumprod) and sch.steps_offset == 1
    sch.set_timesteps(50)
    ref.set_timesteps(50)
    assert torch.equal(sch.timesteps, ref.timesteps)


REFUSED = [("beta_schedule", "linear"), ("beta_schedule", "squaredcos_cap_v2"), ("set_alpha_to_one", True),
           ("clip_sample", True), ("thresholding", True), ("timestep_spacing", "trailing"),
           ("timestep_spacing", "linspace"), ("rescale_betas_zero_snr", True), ("trained_betas", [0.1] * 1000),
           ("prediction_type", "sample")]


@pytest.mark.parametrize("key,value", REFUSED, ids=[f"{k}={v if not isinstance(v, list) else 'list'}"
                                                    for k, v in REFUSED])
def test_from_config_refuses_what_it_does_not_compute(key, value):
    with pytest.raises(ValueError, match=re.escape(key)) as e:
        DDIMScheduler.from_config(dict(SD21_V, **{key: value}))
    if not isinstance(value, list):
        assert repr(value) in str(e.value)


def test_from_config_missing_keys_take_the_diffusers_defaults():
    """diffusers' defaults clip samples and use linear betas: a config that relies on them is refused."""
    for key in ("clip_sample", "beta_schedule", "set_alpha_to_one"):
        with pytest.raises(ValueError, match=key):
            DDIMScheduler.from_config({k: v for k, v in SD21_V.items() if k != key})
    assert DDIMScheduler.from_config({k: v for k, v in SD21_BASE.items() if k != "prediction_type"}).prediction_type \
        == "epsilon"


def test_constructor_defaults_and_refusals():
    assert DDIMScheduler().prediction_type == "epsilon"
    with pytest.raises(ValueError, match="sample"):
        DDIMScheduler(prediction_type="sample")


# ------------------------------------------------------------------------------------------------
# e. a tiny-UNet v edit
# ------------------------------------------------------------------------------------------------
def _edit(world, rank, mode, steps, fused, kind=V):
    from oracle.oracle_ops import OracleOps
    from tokenflow_b200 import sd_unet
    from tokenflow_b200.editor import synthetic_inputs
    tfu._install_ops_for_testing(OracleOps())
    unet = sd_unet.build_unet("tiny", seed=1)
    cfg = {"n_frames": 8, "batch_size": 2, "n_timesteps": steps, "guidance_scale": 7.5, "mode": mode,
           "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "start": 0.9, "fused_pass": fused}
    x, text, pnp, src = synthetic_inputs(8, 16, unet.config.cross_attention_dim, steps, seed=1, ctx_len=7)
    ed = TokenFlowEditor(unet, DDIMScheduler(prediction_type=kind), tfu, cfg, text, pnp,
                         source_latents=lambda t: src[t], world_size=world, rank=rank)
    ed.init_method()
    torch.manual_seed(1)
    return ed.sample_loop(x), ed.keyframe_log


@pytest.mark.parametrize("mode,steps", [("pnp", 2), ("sdedit", 10)])
def test_fused_v_edit_equals_the_reference_schedule(mode, steps):
    ref, kf_ref = _edit(1, 0, mode, steps, fused=False)
    got, kf = _edit(1, 0, mode, steps, fused=True)
    eps, _ = _edit(1, 0, mode, steps, fused=True, kind="epsilon")
    assert kf == kf_ref
    assert torch.allclose(got, ref, atol=2e-4, rtol=1e-4), (got - ref).abs().max().item()
    assert (got - eps).abs().max() > 1e-2                        # the v step is the one that ran


def _worker(rank, world, rdzv, mode, steps, q):
    torch.set_num_threads(2)
    dist.init_process_group("gloo", init_method=f"file://{rdzv}", rank=rank, world_size=world)
    try:
        out, kf = _edit(world, rank, mode, steps, fused=True)
        q.put((rank, out.numpy().tolist(), kf))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("mode,steps", [("pnp", 2), ("sdedit", 10)])
def test_two_rank_v_edit_equals_single_process(mode, steps):
    want, kf_want = _edit(1, 0, mode, steps, fused=False)
    fd, rdzv = tempfile.mkstemp(prefix="tf_b200_vpred_rdzv_")
    os.close(fd)
    os.unlink(rdzv)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, rdzv, mode, steps, q)) for r in range(2)]
    for p in procs:
        p.start()
    results = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, out, kf in results:
        assert kf == kf_want
        assert torch.allclose(torch.tensor(out), want, atol=2e-4, rtol=1e-4), f"rank {rank}"
