"""K2a's twelve-site kernel on pileups whose (strand x base) groups hold no neighbour-mismatch call.  Such a group's dependent error
probabilities come from the clean-group rows of the context's tables (the rank of each member times its quality); groups of up to 16
members are ranked in the grouping phase, larger ones still go through the std::sort mirror.  Every call of a batch has one quality, so
all members of a group tie and the sort's treatment of equal keys decides which call gets which exponent.  Each field is compared
with the oracle bit for bit, at the default exponent parameters and at ones that move the clamp (or never reach it within the rows)."""
import numpy as np
import pytest

import reflib
from strelka_b200 import _abi as A
from strelka_b200 import batch as B

pytestmark = pytest.mark.gpu


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64 if a.dtype == np.float64 else np.uint32)


def _clean_sites(rng, n_sites, q, big):
    """Sites of one or two reference-base groups (forward and reverse strand) and sometimes a small alternative-base group, the
    strands interleaved at random in pileup order.  Group sizes 1-16; when `big`, the first group holds 17-40 calls and half the time
    the second does too, so that sites of more than 64 calls (the kernel's deeper grouping loop) occur.  At most 96 calls."""
    sites, refs = [], []
    for _ in range(n_sites):
        ref = int(rng.integers(0, 4))
        alt = (ref + 1 + int(rng.integers(0, 3))) % 4
        groups = [(ref, 1, int(rng.integers(17, 41)) if big else int(rng.integers(1, 17)))]
        if rng.random() < 0.8:
            groups.append((ref, 0, int(rng.integers(17, 41)) if big and rng.random() < 0.5 else int(rng.integers(1, 17))))
        if rng.random() < 0.3:
            groups.append((alt, int(rng.integers(0, 2)), int(rng.integers(1, 9))))
        calls = [int(B.pack_call(q, base, fwd)) for base, fwd, k in groups for _ in range(k)]
        rng.shuffle(calls)
        sites.append(calls)
        refs.append("ACGT"[ref])
    return B.PileupBatch.from_sites(sites, "".join(refs))


@pytest.mark.parametrize("ssd_no", [None, 0.2, 0.6, 0.05])  # clamp after 4 ranks (defaults), 7, 2; not within the table's 8
@pytest.mark.parametrize("q", [37, 12])
def test_k2a_clean_groups_one_quality(ssd_no, q):
    from strelka_b200.api import Context

    p = A.default_params()
    if ssd_no is not None:
        p.bsnp_ssd_no_mismatch = ssd_no
    rng = np.random.default_rng(4100 + q + int(1000 * (ssd_no or 0)))
    pb = _clean_sites(rng, 3000, q, big=False)
    pb_big = _clean_sites(rng, 3000, q, big=True)
    ctx = Context(0, p)
    try:
        for batch in (pb, pb_big):
            assert int(np.diff(batch.site_off.astype(np.int64)).max()) <= 96
            for always in (True, False):
                want = reflib.ox_germline(p, batch, always)
                got = ctx.site_gl_germline(batch, always)
                for f in ("ref_gt", "is_computed", "n_used_calls", "phredLoghood"):
                    assert np.array_equal(want[f], got[f]), f
                assert np.array_equal(_bits(want["lhood"]), _bits(got["lhood"]))
                assert np.array_equal(_bits(want["strand_bias"]), _bits(got["strand_bias"]))
                for rs in ("genome", "poly"):
                    for f in ("max_gt", "snp_qphred", "max_gt_qphred"):
                        assert np.array_equal(want[rs][f], got[rs][f]), (rs, f)
                    assert np.array_equal(_bits(got[rs]["ref_pprob"]), _bits(want[rs]["ref_pprob"])), (rs, "ref_pprob")
    finally:
        ctx.close()
