"""GPU: the plain persistent split-bf16 GEMM runs its two consumer warpgroups ping-pong (warpgroup j % 2 owns the
CTA's j-th tile), while variant 3 (non-persistent) gives each warpgroup 64 rows of every tile.  Every output element
still sees the same wgmma in the same order, so variant 4 must equal variant 3 bit for bit: with 1, 2 or 3 tiles per
CTA (warpgroup 1 with no tile or one fewer), one k-block or many, BN = 32 / 64 / 128, every operand majorness and
split-K."""
import pytest

from test_gemm_tma_epilogue_gpu import _run

pytestmark = pytest.mark.gpu

# (m, n, k, trans_a, trans_b, split_k); an H100 runs min(#tiles, 132) CTAs of 128 x BN tiles
CASES = [
    (100, 128, 845, False, False, 1),          # 1 tile: warpgroup 1 idle
    (131 * 128 - 5, 128, 64, False, False, 1), # 131 tiles, one each; a single k-block
    (133 * 128, 128, 845, True, True, 1),      # 133 tiles: CTA 0 has two
    (264 * 128, 128, 128, False, False, 1),    # 264 tiles: two per CTA
    (265 * 128 - 60, 128, 40, False, True, 1), # 265 tiles: CTA 0 has three (warpgroup 1 one fewer); k < one block
    (4000, 200, 300, True, False, 1),          # two N tiles per row block
    (133 * 128, 64, 845, False, True, 1),      # BN = 64
    (1000, 48, 64, True, True, 1),             # BN = 64, 16 clipped columns
    (265 * 128 - 1, 20, 200, False, False, 1), # BN = 32, 265 tiles
    (130, 32, 64, True, False, 1),             # BN = 32, second half of the only tile mostly past m
    (300, 128, 4096, False, False, 3),         # split-K: 9 tiles, register epilogue into the workspace
    (845, 256, 8200, True, False, 8),
]


def _case(cuda, m, n, k, ta, tb, sk):
    _run(cuda, m, n, k, ta, tb, ldc=n + (-n) % 4, sk=sk, bias=sk == 1, act="relu" if sk == 1 else "none")


@pytest.mark.parametrize("m,n,k,ta,tb,sk", CASES)
def test_pingpong_matches_variant3(cuda, m, n, k, ta, tb, sk):
    _case(cuda, m, n, k, ta, tb, sk)
