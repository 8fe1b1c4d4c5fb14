"""CPU suite: the multiplier-pipe budget of K1's squaring loop (mont_sqr's owner loop, rsa_square_r32.cuh), read from the
SASS by tools/k1_sass_budget.py.  The wide multiplies are fixed by the algorithm; the other IMADs (carry limbs, carries
turned into values, register copies, ptxas's IMAD.IADD) take multiplier-pipe cycles from them.  No compute."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from k1_sass_budget import budget  # noqa: E402

# One loop trip = two owner steps.  Other IMADs: 115 with ptxas 12.9, plus a margin for the register allocator, whose
# back-edge copies move with small source changes.
WIDE_PER_TRIP = 784
OTHER_IMAD_MAX = 122


def test_squaring_loop_fma_pipe_budget(built):
    sq = budget(os.path.join(ROOT, "bftkv_b200", "libbftq.so"))["squaring"]
    assert sq["imad_wide"] == WIDE_PER_TRIP and sq["imad_wide_x"] == 2 * 337, sq
    assert sq["imad_other"] <= OTHER_IMAD_MAX, sq
    assert sq["fma_cycles"] <= 4 * WIDE_PER_TRIP + 2 * OTHER_IMAD_MAX, sq
