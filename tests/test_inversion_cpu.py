"""CPU tier: the host side of the graphed inversion path — its coefficient tables against the reference's 0-dim fp32
tensor arithmetic, the saved-timestep set over the reference's 500-step grid, and the frame shares of the ranks."""
import pytest
import torch

from oracle import inversion as OI
from tokenflow_b200.preprocess import LatentInverter, inversion_coef_tables, saved_timesteps
from tokenflow_b200.scheduler import DDIMScheduler


@pytest.mark.parametrize("steps", [500, 50, 7])
def test_coefficient_tables_equal_the_reference_fp32_arithmetic_bit_for_bit(steps):
    sch = DDIMScheduler()
    sch.set_timesteps(steps)
    inv, rec = inversion_coef_tables(sch)
    assert inv.dtype == rec.dtype == torch.float32 and inv.shape == rec.shape == (steps, 4)
    for direction, table in (("inversion", inv), ("reconstruction", rec)):
        for i in range(steps):
            want = OI.step_coefficients(sch, direction, i)
            assert all(w.dtype == torch.float32 and w.dim() == 0 for w in want)
            assert torch.equal(table[i], torch.stack(list(want))), (direction, i, table[i], want)
    # the grid ends use final_alpha_cumprod (= alphas_cumprod[0]): the first inversion step, the last reconstruction one
    a0 = sch.final_alpha_cumprod
    assert torch.equal(inv[0, 0], (1 - a0) ** 0.5) and torch.equal(inv[0, 1], 1 / a0 ** 0.5)
    assert torch.equal(rec[-1, 2], a0 ** 0.5) and torch.equal(rec[-1, 3], (1 - a0) ** 0.5)


def test_coefficient_tables_are_not_the_double_precision_ones():
    """The fp32 steps matter: rounding double-precision square roots once differs from the fp32 chain somewhere on
    the 500-step grid (what the eager CPU loop's `_alphas` computes)."""
    sch = DDIMScheduler()
    sch.set_timesteps(500)
    inv, _ = inversion_coef_tables(sch)
    ts_up = [int(t) for t in reversed(sch.timesteps.tolist())]
    a = sch.alphas_cumprod.double()
    dbl = torch.tensor([float((1 - a[t]) ** 0.5) for t in ts_up], dtype=torch.float32)
    assert not torch.equal(inv[:, 3], dbl)


def test_saved_timesteps_over_500_steps_equal_the_reference_loop():
    """Reference preprocess.py:227-229 with its defaults (:345-347): 500 inversion steps, the 50 sampling timesteps
    saved, plus the last one."""
    sch = DDIMScheduler()
    sch.set_timesteps(500)
    toy = DDIMScheduler()
    toy.set_timesteps(50)
    to_save = toy.timesteps                                # get_timesteps(toy, 50, strength=1.0)
    eps_free = lambda x, t, encoder_hidden_states=None: {"sample": torch.zeros_like(x)}
    _, saved = OI.ddim_inversion(eps_free, sch, torch.zeros(1, 1, 1), torch.zeros(1, 1), 1, to_save)
    ts_up = [int(t) for t in reversed(sch.timesteps.tolist())]
    plan = saved_timesteps(ts_up, to_save.tolist())
    assert plan == sorted(saved) and len(plan) == 51
    assert set(plan) == set(to_save.tolist()) | {ts_up[-1]}


@pytest.mark.parametrize("n,world", [(40, 3), (10, 4), (5, 4), (7, 2), (1, 2), (200, 8)])
def test_rank_shares_cover_the_frames_exactly(n, world):
    frames = []
    for rank in range(world):
        inv = LatentInverter.__new__(LatentInverter)
        inv.world_size, inv.rank = world, rank
        lo, hi = inv._local(n)
        frames += list(range(lo, hi))
        assert max(0, hi - lo) <= -(-n // world)           # every share fits the all-gather's padded slot
    assert frames == list(range(n))
