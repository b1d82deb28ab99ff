"""GPU: the 64-column halo conv's tile schedule.  At BN = 64 one warpgroup issues the MMAs and drains tile t into staging tile
t & 1 while a second warpgroup runs the epilogue of tile t-1, keeping its GroupNorm sums over the CTA's tiles and flushing them
every 8 tiles and at the end.  These cases check the same float64 reference as test_contraction_gpu.test_conv3 at the tile
counts where that schedule has edges (H100: 132 SMs, one CTA per SM):

  * fewer tiles than SMs: every CTA runs a single tile, so only staging tile 0 is used and the final flush is the only one;
  * 296 tiles: CTAs run 2 or 3 tiles (an odd count ends on staging tile 0), stats remainder 2 or 3;
  * 1200 tiles: CTAs run 9 or 10 tiles, one 8-tile flush and a remainder of 1 or 2;
  * a drain every tap and every 3 taps at 64 -> 64 channels."""
import pytest

from tests import test_contraction_gpu as TC

pytestmark = pytest.mark.gpu

CASES = [  # path, F, H, W, Cin, N, drain
    ("conv3", 3, 16, 16, 64, 64, 0), ("tma", 3, 16, 16, 64, 64, 0),
    ("conv3", 37, 32, 32, 64, 64, 0), ("tma", 37, 32, 32, 64, 64, 0),
    ("conv3", 150, 32, 32, 64, 64, 0), ("tma", 150, 32, 32, 64, 64, 0),
    ("conv3", 20, 32, 32, 64, 64, 3), ("tma", 20, 32, 32, 64, 64, 1),
    ("conv3", 20, 32, 32, 64, 64, 1), ("tma", 20, 32, 32, 64, 64, 3),
]


@pytest.mark.parametrize("path,F,H,W,Cin,N,drain", CASES,
                         ids=[f"{'gather' if c[0] == 'conv3' else 'tma'}-F{c[1]}-{c[2]}x{c[3]}-{c[4]}-{c[5]}-d{c[6]}" for c in CASES])
def test_conv3_bn64_schedule(path, F, H, W, Cin, N, drain):
    TC.test_conv3(path, F, H, W, Cin, N, drain)
