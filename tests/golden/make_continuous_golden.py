"""Freezes the reference's answers for K2c into tests/golden/continuous_ref.npz (needs oracle/_ref/libstrelka_ref_continuous.so):
  first[n, q-1]  the first a whose getAlleleSequencingErrorQscore(a, n, 17, 40) reaches q, for every n <= 16384 (0xffff where no a <= n
                 does); every a up to min(n, L + 10 sqrt(L) + 40), L = n * 10^-1.7, was evaluated (top[n] is the last), and GQ ascends in a
  top[n]         the last a evaluated at n
  large_a, large_n  sampled pairs past the grid, all GQ 40
  sb_counts, sb_ref  strandBias(fwdAlt, revAlt, fwdOther, revOther) for seeded counts
The same bytes on every run."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import continuous_gen as G  # noqa: E402

a, n = G.grid_pairs()
gq = G.ref_qscore(a, n)
first, top = G.grid_thresholds(a, n, gq)
assert np.all((first[:, 39] <= top) | (top == np.arange(G.GRID_N + 1))), "the grid reaches GQ 40 wherever a <= n can"
la, ln = G.sampled_large_pairs()
assert np.all(G.ref_qscore(la, ln) == 40)
sb_counts = G.strand_bias_cases()
np.savez_compressed(G.GOLDEN, first=first, top=top, large_a=la, large_n=ln, sb_counts=sb_counts, sb_ref=G.ref_strand_bias(sb_counts))
print(f"{len(a)} grid pairs, {len(la)} large pairs, {len(sb_counts)} strand-bias cases -> {G.GOLDEN}")
