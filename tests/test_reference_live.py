"""CPU tier: the oracle against outputs of the UNMODIFIED reference hooks and helpers, recorded on fresh
seeds by oracle/gen_golden.py (`live_cases`) in tests/golden/reference_live.pt."""
import pytest
import torch

from oracle import golden
from oracle import tokenflow_oracle as O
from tokenflow_b200 import sd_unet


@pytest.fixture(scope="module")
def live(golden_dir):
    return golden.load(golden_dir, "reference_live.pt")


@pytest.mark.parametrize("seed,n,S,dim,heads,pnp,inject", [
    (101, 2, 24, 32, 2, False, False), (102, 4, 20, 64, 4, True, True), (103, 4, 20, 64, 4, True, False),
    (104, 13, 8, 32, 4, True, True)])
def test_live_extended_attention(live, seed, n, S, dim, heads, pnp, inject):
    c = live["attn"][seed]
    block = sd_unet.BasicTransformerBlock(dim, heads, dim // heads, 16).eval()
    block.attn1.load_state_dict(c["state_dict"])
    x, want = c["x"], c["out"]
    assert x.shape == (3 * n, S, dim)
    with torch.no_grad():
        a = block.attn1
        got = a.to_out[0](O.extended_attention(a.to_q(x), a.to_k(x), a.to_v(x), heads, a.scale, inject))
    assert torch.allclose(got, want, atol=2e-6, rtol=1e-5)


def test_live_cosine_sim_and_isinstance_str(live):
    from tokenflow_b200.util import isinstance_str
    c = live["cosine"]
    assert torch.equal(O.cosine_sim(c["x"], c["y"]), c["sim"])
    blk = sd_unet.BasicTransformerBlock(16, 2, 8, 8)
    for name, want in live["isinstance_str"].items():
        assert isinstance_str(blk, name) == want
