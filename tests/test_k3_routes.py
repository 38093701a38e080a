"""K3 global_align on every launch route: the group kernel's 64 buckets, the warp kernel's register and shared-memory strips, launches
of 4, 2 and 1 warps per CTA, status 2, and the two entry points -- against the CPU oracle, and the oracle against the reference on
the same shapes and scores.  The routing itself is restated in tests/k3_routes.py; the first test pins that restatement to the
sources."""
import collections
import os
import re

import numpy as np
import pytest

import k3_routes as K
import reflib
from strelka_b200 import _abi as A
from strelka_b200 import batch as B

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "strelka_b200", "csrc")
STATUS2 = (0, 0, 0, 2)
POISON = 0xA5A5A5A5


def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _pool(batches):
    return [p for pairs in batches.values() for p in pairs]


def _ga_batch(pairs, max_ops=None):
    if max_ops is None:  # an alignment has at most Q + R operations: no overflow
        max_ops = max(len(q) + len(r) for q, r in pairs) + 2
    return B.GaBatch([q for q, _ in pairs], [r for _, r in pairs], max_ops=max_ops)


# ---------------------------------------------------------------------------------------------------------------------------------
# CPU: the mirror and the cases
# ---------------------------------------------------------------------------------------------------------------------------------
def test_route_constants_match_the_strip_and_slot_sources():
    """Every constant tests/k3_routes.py copies, read back out of the kernels -- the routing constants, the four register-strip
    instantiations and every term of the warp kernel's slot layout: a routing change must update the mirror (and with it the route
    matrix the other tests check) in the same commit."""
    grp, warp, common = _src("k3_group.cu"), _src("k3_global_align.cu"), _src("k3_common.cuh")
    m = re.search(r"constexpr uint32_t KG_MAX_Q = (\d+), KG_MAX_R = (\d+);", grp)
    assert m and (int(m[1]), int(m[2])) == (K.KG_MAX_Q, K.KG_MAX_R)
    assert int(re.search(r"constexpr int KG_G = (\d+);", grp)[1]) == K.KG_G
    assert int(re.search(r"constexpr int KG_RCLASSES = (\d+);", grp)[1]) == K.KG_RCLASSES
    assert re.search(r"return \(T - 1\) \* KG_RCLASSES \+ min\(\(uint32_t\)KG_RCLASSES - 1, R >> 6\);", grp)
    assert re.search(r"if \(Q == 0 \|\| R == 0 \|\| Q > max_q \|\| R > KG_MAX_R\) return KG_BUCKETS - 1;", grp)
    m = re.search(r"const auto big = \[\]\(int v\) \{ return v > (\d+) \|\| v < -(\d+); \};", grp)
    assert m and int(m[1]) == int(m[2]) == K.KG_SCORE_MAX
    fields = re.search(r"const uint32_t max_q = \(([^?]*)\) \? 0u : KG_MAX_Q;", grp)[1]
    assert re.findall(r"big\(sc->(\w+)\)", fields) == list(K.SCORE_FIELDS)
    assert int(re.search(r"constexpr int K3_WARPS = (\d+);", warp)[1]) == K.K3_WARPS
    assert "while (warps > 1 && slot * warps > ctx->smem_optin) warps >>= 1;" in warp
    assert "if (Q == 0 || R == 0 || k3_slot_bytes(Q, R) > slot_bytes)" in warp
    assert re.findall(r"case (\d): dp_register_strip<\1>\(", warp) == ["1", "2", "3", "4"]
    assert "default: dp_shared_strip(" in warp
    assert "uint32_t k3_slot_bytes(uint32_t Q, uint32_t R) { return k3_slot(Q, R).bytes; }" in common
    body = re.search(r"k3_slot_layout k3_slot\(uint32_t Q, uint32_t R\)\s*\{(.*?)\n\}", common, re.S)[1]
    assert re.search(r"s\.bytes = o;\s*return s;\s*$", body)
    terms = [re.sub(r"\s+", "", t) for t in re.findall(r"o \+= ([^;]+);", body)]
    assert re.search(r"const uint32_t T = \(Q \+ 31\) / 32;", body)
    assert terms == ["pad16u((Q+1)*(R+1))", "3u*32u*T*4u", "pad16u(Q+8)", "pad16u(R+8)", "pad16u(Q+R+8)"], terms


def test_route_mirror_on_known_shapes():
    o, sc = K.H100_SMEM_OPTIN, K.score_set("active_region-ins1-del1")
    assert K.k3_route(1023, 211, sc, o) == ("warp_smem", 32) and K.k3_route(1023, 212, sc, o) == "status2"
    assert K.k3_route(128, 255, sc, o) == ("group", 16, 3) and K.k3_route(128, 256, sc, o) == ("warp_reg", 4)
    assert K.k3_route(129, 10, sc, o) == ("warp_smem", 5) and K.k3_route(0, 5, sc, o) == "empty"
    assert K.k3_route(64, 64, K.score_set("open-4097-ins0-del0"), o) == ("warp_reg", 2)
    assert K.k3_route(64, 64, K.score_set("open-4096-ins0-del0"), o) == ("group", 8, 1)
    assert K.k3_warp_launch_warps([(10, 10)], sc, o) is None
    assert K.k3_warp_launch_warps([(128, 300), (10, 10)], sc, o) == 4
    assert K.k3_warp_launch_warps([(128, 511)], sc, o) == 2
    assert K.k3_warp_launch_warps([(128, 1000), (1023, 212)], sc, o) == 1


def test_active_region_scores_are_a_case_score_set():
    s = A.SxGaScores()
    A.load().sx_ga_active_region_scores(s)
    assert bytes(s) == bytes(K.score_set("active_region-ins1-del1"))


def test_cases_reach_every_route():
    """The cases fill every route with several problems: all 64 group buckets, register strips T = 1..4 (with DP row Q in the last
    row of the strip and, for T > 1, above it), shared-memory strips T = 5..32, status 2, and warp launches of 4, 2 and 1 warps."""
    o = K.H100_SMEM_OPTIN
    sc = K.score_set("active_region-ins1-del1")
    batches = K.route_batches(o)
    count = collections.Counter()
    r_last = collections.Counter()
    for pairs in batches.values():
        for q, r in pairs:
            rt = K.k3_route(len(q), len(r), sc, o)
            count[rt] += 1
            if K.route_kind(rt) == "warp_reg":
                r_last[(rt[1], K.reg_strip_r_last(len(q)) == rt[1] - 1)] += 1
    # the register strips also run the group-kernel shapes once a score is past +-4096
    big = K.score_set("open-4097-ins0-del0")
    for q, r in batches["group"]:
        rt = K.k3_route(len(q), len(r), big, o)
        assert K.route_kind(rt) == "warp_reg"
        r_last[(rt[1], K.reg_strip_r_last(len(q)) == rt[1] - 1)] += 1
    want = [("group", t, c) for t in range(1, 17) for c in range(4)] + [("warp_reg", t) for t in range(1, 5)]
    want += [("warp_smem", t) for t in range(5, 33)] + ["status2"]
    few = {k: count[k] for k in want if count[k] < 3}
    assert not few, few
    assert set(count) == set(want)
    assert r_last[(1, True)] >= 3 and r_last[(1, False)] == 0  # one row per lane: always the last
    assert all(r_last[(t, True)] >= 3 and r_last[(t, False)] >= 3 for t in (2, 3, 4)), r_last
    warps = {name: K.k3_warp_launch_warps(K.shapes_of(p), sc, o) for name, p in batches.items()}
    assert warps == {"group": None, "warp4": 4, "warp2": 2, "warp1": 1}
    kinds = collections.Counter(K.route_kind(k) for k in count.elements())
    print(f"problems per route: {dict(kinds)}; per key: {dict(sorted(count.items(), key=str))}")
    # the cases differ from one run to the next only if the generator changes
    assert K.route_batches(o) == batches


# ---------------------------------------------------------------------------------------------------------------------------------
# CPU: the oracle against the reference on the same routes
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.ref
@pytest.mark.parametrize("base", list(K.BASE_SCORES))
def test_oracle_matches_reference_on_every_route(base):
    """oracle/strelka_oracle.cpp against GlobalAligner<int> on one problem of every route each score set gives (status-2 shapes
    included: the reference has no size limit), all four flag combinations; records and cigar rows byte for byte, with room for
    every operation and with max_ops 0 and 3."""
    pool = _pool(K.route_batches())
    for f, (ins, dele) in enumerate(K.FLAGS):
        sc = K.ga_scores(*K.BASE_SCORES[base], ins, dele)
        pairs = K.route_sample(pool, sc, K.H100_SMEM_OPTIN, 1, seed=4 * list(K.BASE_SCORES).index(base) + f)
        kinds = {K.route_kind(K.k3_route(len(q), len(r), sc, K.H100_SMEM_OPTIN)) for q, r in pairs}
        assert kinds >= {"warp_reg", "warp_smem", "status2"}
        small = [(q, r) for q, r in pairs if len(q) * len(r) <= 20000]
        for max_ops, sub in ((None, pairs), (0, small), (3, small)):
            gb = _ga_batch(sub, max_ops)
            r_res, r_cig = reflib.ref_global_align(sc, gb)
            o_res, o_cig = reflib.ox_global_align(sc, gb)
            assert r_res.tobytes() == o_res.tobytes(), (base, ins, dele, max_ops)
            assert r_cig.tobytes() == o_cig.tobytes(), (base, ins, dele, max_ops)


# ---------------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ctx():
    from strelka_b200.api import Context

    c = Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def optin():
    import torch

    return int(torch.cuda.get_device_properties(0).shared_memory_per_block_optin)


@pytest.fixture(scope="module")
def batches(optin):
    return K.route_batches(optin)


def _expected(sc, pairs, gb, optin):
    """the oracle's records and rows, with what the device returns for a problem too large for a slot: {0, 0, 0, 2} and a row the
    kernel did not write"""
    res, cig = reflib.ox_global_align(sc, gb)
    s2 = np.array([K.k3_route(len(q), len(r), sc, optin) == "status2" for q, r in pairs], bool)
    res[s2] = STATUS2
    cig[s2] = 0
    return res, cig


def _assert_same(got, want, pairs, sc, optin, what):
    (g_res, g_cig), (w_res, w_cig) = got, want
    bad = np.nonzero((g_res != w_res) | np.any(g_cig != w_cig, axis=1))[0]
    if bad.size:
        i = int(bad[0])
        q, r = pairs[i]
        raise AssertionError(f"{what}: {bad.size} of {len(pairs)} problems differ; first: #{i} Q={len(q)} R={len(r)} "
                             f"route={K.k3_route(len(q), len(r), sc, optin)} got {g_res[i]} {B.cigar_string(g_cig[i][: min(g_res[i]['n_ops'], g_cig.shape[1])])} "
                             f"want {w_res[i]} {B.cigar_string(w_cig[i][: min(w_res[i]['n_ops'], w_cig.shape[1])])}")


def _run_dev(ctx, sc, gb):
    """sx_global_align_dev with its record and cigar buffers filled with 0xA5 first"""
    from strelka_b200.api import DevGaBatch

    db = DevGaBatch(ctx, gb)
    db.res.upload(np.full(db.res.nbytes, 0xA5, np.uint8))
    db.cigar.upload(np.full(db.cigar.nbytes, 0xA5, np.uint8))
    ctx.global_align_dev(sc, db)
    res = db.res.download(A.GA_RESULT_DT, gb.n)
    cig = db.cigar.download(np.uint32, db.cigar.nbytes // 4)
    for b in list(db.bufs.values()) + [db.res, db.cigar]:
        b.free()
    return res, cig


FULL_BATCH_BASES = ("active_region", "golden")


@pytest.mark.gpu
@pytest.mark.parametrize("sid", K.score_set_ids())
def test_host_entry_matches_oracle_on_every_route(ctx, optin, batches, sid):
    """sx_global_align == the oracle, byte for byte, on each case batch (the whole batches for the production and the golden scores,
    two problems of every route for the others); status-2 problems come back as {0, 0, 0, 2} with a zero row."""
    sc = K.score_set(sid)
    for name, pairs in batches.items():
        if sid.rsplit("-", 2)[0] not in FULL_BATCH_BASES:
            pairs = K.route_sample(pairs, sc, optin, 2, seed=K.score_set_ids().index(sid))
        gb = _ga_batch(pairs)
        _assert_same(ctx.global_align(sc, gb), _expected(sc, pairs, gb, optin), pairs, sc, optin, f"{sid} {name}")


@pytest.mark.gpu
@pytest.mark.parametrize("sid", ["active_region-ins1-del1", "golden-ins0-del0", "open-4097-ins1-del0"])
def test_device_entry_matches_host_entry(ctx, optin, batches, sid):
    """sx_global_align_dev on the same batches, plus empty queries and references: the host entry's records, the first
    min(n_ops, max_ops) words of each cigar row, and every other word of the (0xA5-filled) buffers untouched; status-2 and empty
    problems get {0, 0, 0, 2} and leave their row alone."""
    sc = K.score_set(sid)
    empties = [("", "ACGT"), ("ACGTA", ""), ("", "")]
    for name, pairs in batches.items():
        if name == "warp1" and not sid.startswith("active"):
            pairs = K.route_sample(pairs, sc, optin, 3, seed=5)
        gb = _ga_batch(pairs)
        h_res, h_cig = ctx.global_align(sc, gb)
        mixed = pairs[:7] + empties + pairs[7:]
        n, mo = len(mixed), gb.max_ops
        d_res, d_words = _run_dev(ctx, sc, _ga_batch(mixed, mo))
        d_cig, tail = d_words[: n * mo].reshape(n, mo), d_words[n * mo :]
        want_res = np.concatenate([h_res[:7], np.array([STATUS2] * len(empties), A.GA_RESULT_DT), h_res[7:]])
        want_cig = np.concatenate([h_cig[:7], np.zeros((len(empties), mo), np.uint32), h_cig[7:]])
        assert d_res.tobytes() == want_res.tobytes(), (sid, name)
        for i in range(n):
            k = min(int(want_res["n_ops"][i]), mo) if want_res["status"][i] != 2 else 0
            assert np.array_equal(d_cig[i, :k], want_cig[i, :k]), (sid, name, i)
            assert np.all(d_cig[i, k:] == POISON), (sid, name, i, len(mixed[i][0]), len(mixed[i][1]))
        assert np.all(tail == POISON)


def _overflow_problems(batches, sc, optin):
    """register-strip, shared-strip and T = 16 group problems with at least 7 operations"""
    pick = []
    for pairs in batches.values():
        for q, r in pairs:
            rt = K.k3_route(len(q), len(r), sc, optin)
            if K.route_kind(rt) in ("warp_reg", "warp_smem") or rt[:2] == ("group", 16):
                pick.append((q, r))
    res, _ = reflib.ox_global_align(sc, _ga_batch(pick))
    rng = np.random.default_rng(3)
    out = collections.defaultdict(list)
    for (q, r), n_ops in zip(pick, res["n_ops"]):
        if n_ops >= 7:
            out[K.route_kind(K.k3_route(len(q), len(r), sc, optin))].append((q, r, int(n_ops)))
    return {k: [v[i] for i in rng.permutation(len(v))[:6]] for k, v in out.items()}


@pytest.mark.gpu
def test_cigar_overflow_on_every_kernel(ctx, optin, batches):
    """max_ops of 1, 2, 3, 5, n_ops - 1 and n_ops on the register strips, the shared-memory strips and the T = 16 group kernel:
    status 1 exactly when n_ops > max_ops, n_ops the true count, and the first max_ops operations in the row."""
    sc = K.score_set("golden-ins1-del0")
    probs = _overflow_problems(batches, sc, optin)
    assert set(probs) == {"warp_reg", "warp_smem", "group"} and all(len(v) >= 4 for v in probs.values()), {k: len(v) for k, v in probs.items()}
    flat = [p for v in probs.values() for p in v]
    full, full_cig = reflib.ox_global_align(sc, _ga_batch([(q, r) for q, r, _ in flat]))
    runs = [(mo, flat) for mo in (1, 2, 3, 5)] + [(n + d, [p]) for p in flat for n in [p[2]] for d in (-1, 0)]
    for mo, sub in runs:
        pairs = [(q, r) for q, r, _ in sub]
        gb = _ga_batch(pairs, mo)
        g_res, g_cig = ctx.global_align(sc, gb)
        _assert_same((g_res, g_cig), reflib.ox_global_align(sc, gb), pairs, sc, optin, f"max_ops={mo}")
        for i, (q, r, n_ops) in enumerate(sub):
            j = flat.index(sub[i])
            assert g_res["n_ops"][i] == n_ops and g_res["status"][i] == (1 if n_ops > mo else 0)
            assert np.array_equal(g_cig[i, : min(mo, n_ops)], full_cig[j, : min(mo, n_ops)])


@pytest.mark.gpu
def test_max_ops_zero_on_both_kernels_and_entries(ctx, optin, batches):
    """max_ops == 0: every problem reports status 1 and its true operation count, and no cigar word is written (group kernel and
    warp kernel, host entry and device entry)."""
    sc = K.score_set("active_region-ins1-del1")
    pairs = [p for v in batches.values() for p in K.route_sample(v, sc, optin, 2, seed=9)]
    kinds = {K.route_kind(K.k3_route(len(q), len(r), sc, optin)) for q, r in pairs}
    assert kinds == {"group", "warp_reg", "warp_smem", "status2"}
    want, _ = _expected(sc, pairs, _ga_batch(pairs, 0), optin)
    assert np.all((want["status"] == 1) | (want["status"] == 2)) and np.all(want["n_ops"][want["status"] == 1] > 0)
    gb = _ga_batch(pairs, 0)
    g_res, g_cig = ctx.global_align(sc, gb)
    assert g_res.tobytes() == want.tobytes() and g_cig.shape == (len(pairs), 0)
    d_res, d_words = _run_dev(ctx, sc, gb)
    assert d_res.tobytes() == want.tobytes()
    assert np.all(d_words == POISON)


@pytest.mark.gpu
def test_results_do_not_depend_on_the_batch(ctx, optin, batches):
    """The same problems alone, inside a batch whose warp launch runs 4 warps per CTA, and inside the mixed batch that drops it to 1:
    identical records and rows."""
    sc = K.score_set("offedge1-ins1-del0")
    sample = K.route_sample(batches["warp4"], sc, optin, 2, seed=11)
    assert {K.route_kind(K.k3_route(len(q), len(r), sc, optin)) for q, r in sample} == {"group", "warp_reg", "warp_smem"}
    four, one = batches["warp4"], batches["warp1"] + sample
    assert K.k3_warp_launch_warps(K.shapes_of(four), sc, optin) == 4 and K.k3_warp_launch_warps(K.shapes_of(one), sc, optin) == 1
    mo = max(len(q) + len(r) for q, r in four + one) + 2
    alone = [ctx.global_align(sc, _ga_batch([p], mo)) for p in sample]
    a_res = np.concatenate([a[0] for a in alone])
    a_cig = np.concatenate([a[1] for a in alone])
    f_res, f_cig = ctx.global_align(sc, _ga_batch(four, mo))
    idx = [four.index(p) for p in sample]
    o_res, o_cig = ctx.global_align(sc, _ga_batch(one, mo))
    tail = slice(len(one) - len(sample), len(one))
    assert a_res.tobytes() == f_res[idx].tobytes() == o_res[tail].tobytes()
    assert a_cig.tobytes() == f_cig[idx].tobytes() == o_cig[tail].tobytes()
    _assert_same((a_res, a_cig), _expected(sc, sample, _ga_batch(sample, mo), optin), sample, sc, optin, "alone")


@pytest.mark.gpu
@pytest.mark.parametrize("field", ["open", "offedge", "match"])
def test_score_limit_of_the_group_kernel(ctx, optin, batches, field):
    """The group-kernel shapes with one score at the limit (+-4096: group kernel) and one past it (+-4097: the warp kernel's register
    strips), each against the oracle."""
    pairs = batches["group"]
    for base in ([f"{field}-4096", f"{field}-4097"] if field != "match" else ["match+4096", "match+4097"]):
        for ins, dele in ((True, True), (False, False)):
            sc = K.ga_scores(*K.BASE_SCORES[base], ins, dele)
            kinds = {K.route_kind(K.k3_route(len(q), len(r), sc, optin)) for q, r in pairs}
            assert kinds == ({"group"} if base.endswith("4096") else {"warp_reg"})
            gb = _ga_batch(pairs)
            _assert_same(ctx.global_align(sc, gb), _expected(sc, pairs, gb, optin), pairs, sc, optin, base)


@pytest.mark.gpu
def test_host_entry_rejects_empty_problems(ctx, batches):
    """An empty query or reference is an argument error of the host entry (GlobalAligner asserts on it), and the context keeps
    working afterwards."""
    from strelka_b200.api import SxError

    sc = K.score_set("active_region-ins1-del1")
    good = batches["warp4"][:20]
    for bad in (("", "ACGT"), ("ACGT", ""), ("", "")):
        with pytest.raises(SxError) as e:
            ctx.global_align(sc, _ga_batch(good[:5] + [bad] + good[5:]))
        assert e.value.code == A.SX_ERR_ARG
    gb = _ga_batch(good)
    got = ctx.global_align(sc, gb)
    want = reflib.ox_global_align(sc, gb)
    assert got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes()
