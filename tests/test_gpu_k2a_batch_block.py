"""K2a's twelve-site kernel takes each batch's calls as one block: staged from the 16-byte boundary below the block, filtered and grouped
32 calls at a time across site boundaries, with per-(site, group) counts carried from chunk to chunk.  These pileups put site and group
boundaries where that bookkeeping can go wrong; every result field is compared with the oracle, bit for bit where the reference is float."""
import numpy as np
import pytest

import reflib
from strelka_b200 import _abi as A
from strelka_b200 import batch as B

pytestmark = pytest.mark.gpu

# q < 3 as 1 and 2: at q = 0 ln(1 - eprob) is -inf, and a strand bias of -inf - -inf is a NaN whose bits differ between the host and the GPU
QS = np.array([1, 2, 3, 4, 11, 17, 25, 30, 37, 40, 41, 60], np.uint16)


@pytest.fixture(scope="module")
def ctx():
    from strelka_b200.api import Context

    c = Context(0)
    yield c
    c.close()


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64 if a.dtype == np.float64 else np.uint32)


def _same_germline(want, got):
    for f in ("ref_gt", "is_computed", "n_used_calls", "phredLoghood"):
        assert np.array_equal(want[f], got[f]), f
    assert np.array_equal(_bits(want["lhood"]), _bits(got["lhood"]))
    assert np.array_equal(_bits(want["strand_bias"]), _bits(got["strand_bias"]))
    for rs in ("genome", "poly"):
        for f in ("max_gt", "snp_qphred", "max_gt_qphred"):
            assert np.array_equal(want[rs][f], got[rs][f]), (rs, f)
        assert np.array_equal(_bits(got[rs]["ref_pprob"]), _bits(want[rs]["ref_pprob"])), (rs, "ref_pprob")


def _random_site(rng, n, ref_id, filt_frac=0.05, nbr_frac=0.1, odd_frac=0.0):
    """n calls: mostly the reference base, some alt calls, the quality mix includes q < 3.  odd_frac: calls with a base id of 4-15, which
    no pile-up of the reference holds (snp_util.hh asserts it) and whose likelihood terms are undefined there (digt_expect2 reads past its
    table): only at sites whose reference is N, which are filtered and counted but not genotyped"""
    alt = (ref_id + int(rng.integers(1, 4))) % 4
    base = np.where(rng.random(n) < float(rng.choice([0.0, 0.1, 0.5])), alt, ref_id)
    odd = rng.random(n) < odd_frac
    base[odd] = rng.integers(4, 16, int(odd.sum()))
    return B.pack_call(rng.choice(QS, n), base, rng.random(n) < 0.5, rng.random(n) < nbr_frac, rng.random(n) < filt_frac).tolist()


def _edge_sites(rng):
    """(calls, reference base) of sites that sit on the chunk and group edges"""
    sites = [([], "A"), ([], "G"), ([int(B.pack_call(30, 1, 1, filt=1))] * 5, "C"), (B.pack_call(rng.choice(QS, 40), 2, 1, filt=1).tolist(), "G")]
    for n in (31, 32, 33, 63, 64, 65, 95, 96):
        ref = int(rng.integers(0, 4))
        sites.append((_random_site(rng, n, ref, filt_frac=0.0 if n % 2 else 0.05), "ACGT"[ref]))
    # one (site, group) whose members straddle two and three 32-call chunks: one strand and base, q >= 3, a few calls of other groups between
    for n in (60, 96):
        calls = B.pack_call(rng.choice(QS[2:], n), 0, 1).tolist()
        for i in rng.choice(n, 6, replace=False):
            calls[i] = int(B.pack_call(25, int(rng.integers(1, 4)), 0))
        sites.append((calls, "A"))
    # neighbour-mismatch calls in one group only (rev-strand T), the other groups clean
    calls = B.pack_call(rng.choice(QS[2:], 70), rng.integers(0, 4, 70), rng.random(70) < 0.5).tolist()
    for i in range(70):
        if ((calls[i] >> 6) & 15) == 3 and not ((calls[i] >> 10) & 1):
            calls[i] |= 1 << 11
    sites.append((calls, "T"))
    # q < 3 calls only (no group); base ids >= 4 only, and mixed with 0-3 (reference N, see _random_site)
    sites.append((B.pack_call(rng.integers(1, 3, 50), rng.integers(0, 4, 50), rng.random(50) < 0.5).tolist(), "C"))
    sites.append((B.pack_call(rng.choice(QS, 45), rng.integers(4, 16, 45), rng.random(45) < 0.5).tolist(), "N"))
    sites.append((_random_site(rng, 70, 0, odd_frac=0.3), "N"))
    return sites


def _batch(rng, n_sites, edges=True):
    sites = _edge_sites(rng) if edges else []
    while len(sites) < n_sites:
        n = int(min(96, rng.poisson(float(rng.choice([3.0, 30.0, 60.0])))))
        ref = int(rng.integers(0, 4))
        if rng.random() < 0.02:
            sites.append((_random_site(rng, n, ref, odd_frac=0.2), "N"))
        else:
            sites.append((_random_site(rng, n, ref), "ACGT"[ref]))
    sites = [sites[i] for i in rng.permutation(len(sites))][:n_sites]
    ploidy = np.where(rng.random(len(sites)) < 0.2, 1, 2).astype(np.uint8)
    return B.PileupBatch.from_sites([c for c, _ in sites], "".join(r for _, r in sites), ploidy)


@pytest.mark.parametrize("seed,n_sites", [(0, 1207), (1, 600), (2, 2405)])
@pytest.mark.parametrize("always", [True, False])
def test_k2a_batch_block_edges(ctx, seed, n_sites, always):
    rng = np.random.default_rng(4200 + seed)
    pb = _batch(rng, n_sites)
    depth = np.diff(pb.site_off.astype(np.int64))
    assert depth.max() <= 96  # the twelve-site kernel's route
    for n in (0, 31, 32, 33, 63, 64, 65, 95, 96):
        assert (depth == n).any(), n
    assert len({int(pb.site_off[s]) % 8 for s in range(0, n_sites, 12)}) == 8  # every start of a block inside a 16-byte word
    assert (pb.ploidy == 1).any() and (pb.ploidy == 2).any()
    _same_germline(reflib.ox_germline(A.default_params(), pb, always), ctx.site_gl_germline(pb, always))


@pytest.mark.parametrize("n_sites", [1, 5, 11, 13, 25])
def test_k2a_batch_block_short_batches(ctx, n_sites):
    """fewer than twelve sites, and a last batch of one"""
    rng = np.random.default_rng(4300 + n_sites)
    pb = _batch(rng, n_sites, edges=n_sites >= 13)
    p = A.default_params()
    for always in (True, False):
        _same_germline(reflib.ox_germline(p, pb, always), ctx.site_gl_germline(pb, always))


@pytest.mark.parametrize("depth", [50, 66])
def test_k2a_batch_block_every_site_deepest(ctx, depth):
    """every site as deep as the deepest: a block and its unaligned ends need more slots than the 12 sites' order arrays"""
    rng = np.random.default_rng(4350 + depth)
    refs = rng.integers(0, 4, 12 * 30 + 5)
    pb = B.PileupBatch.from_sites([_random_site(rng, depth, int(r)) for r in refs], "".join("ACGT"[r] for r in refs),
                                  np.where(rng.random(len(refs)) < 0.2, 1, 2).astype(np.uint8))
    p = A.default_params()
    for always in (True, False):
        _same_germline(reflib.ox_germline(p, pb, always), ctx.site_gl_germline(pb, always))


def test_k2a_batch_block_device_route(ctx):
    """the device entry point sizes the staging region from the device's largest twelve-site block; the same sites again behind one
    unused call, so that every block starts 2 bytes further into its 16-byte word"""
    from strelka_b200.api import DeviceArray, DevPileupBatch

    rng = np.random.default_rng(4400)
    pb = _batch(rng, 3001)
    shifted = B.PileupBatch(pb.site_off + 1, np.concatenate([np.zeros(1, np.uint16), pb.calls]), pb.ref_base, pb.ploidy)
    p = A.default_params()
    want = reflib.ox_germline(p, pb, True)
    for batch in (pb, shifted):
        db = DevPileupBatch(ctx, batch)
        out = DeviceArray(ctx, batch.n_sites * A.DIGT_RESULT_DT.itemsize)
        ctx.site_gl_germline_dev(db, out, True)
        got = out.download(A.DIGT_RESULT_DT, batch.n_sites)
        _same_germline(want, got)
