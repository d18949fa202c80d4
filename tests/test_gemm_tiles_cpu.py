"""The tile sq_gemm picks for the Llama-2 7B / 13B verify shapes (no GPU needed: the choice is host arithmetic, for 132
SMs where no device is present): never a cluster of more than 2 CTAs, split-K on the deep ring, and the tiles the
runner's routes were measured at (DESIGN §4)."""
import pytest

from sequoia_b200 import model, ops

# (N, K, flags) -> picked (BN, split, mc)
PICKED = {
    (12288, 4096, 0): (128, 1, 2),                  # 7B q/k/v
    (4096, 4096, 0): (64, 2, 1),                    # 7B o_proj
    (22016, 4096, ops.GEMM_SWIGLU): (192, 1, 1),    # 7B gate_up, SwiGLU fused
    (4096, 11008, 0): (64, 2, 1),                   # 7B down_proj
    (32000, 4096, 0): (256, 1, 1),                  # 7B lm_head
    (27648, 5120, ops.GEMM_SWIGLU): (256, 1, 2),    # 13B gate_up, SwiGLU fused
}


@pytest.mark.parametrize("shape", list(PICKED), ids=lambda s: f"N{s[0]}_K{s[1]}_f{s[2]}")
def test_picked_tiles(shape):
    assert ops.gemm_pick_tiles(*shape) == PICKED[shape]


@pytest.mark.parametrize("N,K", [(n, k) for n in (4096, 5120, 8192, 12288, 15360, 22016, 27648, 32000)
                                 for k in (4096, 5120, 11008, 13824)])
def test_clusters_of_at_most_two_ctas(N, K):
    bn, split, mc = ops.gemm_pick_tiles(N, K)
    assert split * mc <= 2, (N, K, bn, split, mc)


def test_verify_plans_name_the_picked_7b_tiles():
    """The runner routes a projection only at the tile it was measured at: for the 7B, that tile is the one picked."""
    shapes = {"wqkv": (12288, 4096), "wo": (4096, 4096), "wd": (4096, 11008)}
    assert model.VERIFY_PLANS
    for k, tile in model.VERIFY_PLANS.items():
        assert ops.gemm_pick_tiles(*shapes[k])[:2] == tile, k
