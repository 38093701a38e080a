"""CPU: the oracle against the reference's committed golden vectors, and the libm / std::sort mirrors against the live
libm / libstdc++ (the mirrors are what the DEVICE code executes; the oracle itself calls the real functions)."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import reflib
import specgen
from strelka_b200 import _abi as A
from strelka_b200 import batch as B

HERE = os.path.dirname(os.path.abspath(__file__))


def test_oracle_global_aligner_goldens():
    gold = json.load(open(os.path.join(HERE, "golden", "global_aligner_goldens.json")))
    assert len(gold["cases"]) == 22
    for case in gold["cases"]:
        sc = A.SxGaScores(*[int(x) for x in case["scores"]])
        gb = B.GaBatch([case["query"]], [case["ref"]], max_ops=64)
        res, cig = reflib.ox_global_align(sc, gb)
        assert B.cigar_string(cig[0, : res["n_ops"][0]]) == case["cigar"], case["name"]
        assert int(res["beginPos"][0]) == case["beginPos"], case["name"]
        if "score" in case:
            assert int(res["score"][0]) == case["score"], case["name"]


def test_oracle_score_fixture():
    """Frozen outputs of the reference's scoreCandidateAlignment (tests/golden/make_fixtures.py)."""
    fx = np.load(os.path.join(HERE, "golden", "k1_fixture.npz"), allow_pickle=False)
    rng = np.random.default_rng(int(fx["seed"]))
    regions = [specgen.random_region(rng, n_reads=int(rng.integers(1, 8))) for _ in range(int(fx["n_regions"]))]
    batch = B.build_align_batch(regions)
    got = reflib.ox_score(batch)
    assert np.array_equal(got.view(np.uint64), fx["lnp_bits"])


def test_oracle_site_fixtures():
    fx = np.load(os.path.join(HERE, "golden", "k2_fixture.npz"), allow_pickle=False)
    rng = np.random.default_rng(int(fx["seed"]))
    pb = specgen.random_pileups(rng, int(fx["n_sites"]), depth=30.0)
    got = reflib.ox_germline(A.default_params(), pb, True)
    assert np.array_equal(got["phredLoghood"], fx["germ_pl"])
    assert np.array_equal(got["lhood"].view(np.uint32), fx["germ_lhood_bits"])
    assert np.array_equal(got["genome"]["snp_qphred"], fx["germ_snp_q"])
    assert np.array_equal(got["genome"]["max_gt"], fx["germ_max_gt"])
    npb = specgen.random_pileups(rng, int(fx["n_sites"]), depth=30.0, alt_frac_choices=(0.0, 0.0, 0.0, 0.0, 0.02, 0.5))
    tpb0 = specgen.random_pileups(rng, int(fx["n_sites"]), depth=60.0, alt_frac_choices=(0.0, 0.0, 0.05, 0.1, 0.2, 0.4))
    tpb = B.PileupBatch(tpb0.site_off, tpb0.calls, npb.ref_base)
    s = reflib.ox_somatic(A.default_params(), npb, tpb)
    assert np.array_equal(s["is_computed"], fx["som_computed"])
    assert np.array_equal(s["qphred"], fx["som_qss"])
    assert np.array_equal(s["from_ntype_qphred"], fx["som_qss_nt"])
    assert np.array_equal(s["ntype"], fx["som_ntype"])


def test_logf_mirror_matches_libm():
    lib = reflib.oracle()
    libm = C.CDLL("libm.so.6")
    libm.logf.restype = C.c_float
    libm.logf.argtypes = [C.c_float]
    rng = np.random.default_rng(0)
    xs = np.concatenate([rng.integers(0x00800000, 0x7F800000, 200000, dtype=np.int64).astype(np.uint32).view(np.float32),
                         (10.0 ** (-np.arange(0, 71) / 10.0)).astype(np.float32), rng.random(100000, dtype=np.float32) + np.float32(1e-7)])
    for x in xs[:: max(1, len(xs) // 60000)]:
        a = np.float32(libm.logf(float(x)))
        b = np.float32(lib.ox_logf_restated(float(x)))
        assert a.view(np.uint32) == b.view(np.uint32), x


def test_powf_mirror_matches_libm():
    lib = reflib.oracle()
    libm = C.CDLL("libm.so.6")
    libm.powf.restype = C.c_float
    libm.powf.argtypes = [C.c_float, C.c_float]
    rng = np.random.default_rng(1)
    for q in range(3, 71):
        e = np.float32(10.0 ** (-q / 10.0))
        for y in np.concatenate([rng.uniform(0.2, 1.0, 400).astype(np.float32), np.float32([1.0, 0.25, 0.65, 0.4225])]):
            a = np.float32(libm.powf(float(e), float(y)))
            b = np.float32(lib.ox_powf_restated(float(e), float(y)))
            assert a.view(np.uint32) == b.view(np.uint32), (q, y)


def test_double_libm_mirrors_match_libm():
    """sx_exp / sx_log10 / sx_log / sx_log1p (strelka_b200/csrc/sx_libm_mirror_d.h: what the double epilogues of K2a, K2b and K5 execute on the device) give the bits of
    the libm the reference is linked against: normalizeLogDistro's exp(x - max) over its whole range incl. the subnormal results and the
    underflow to 0, error_prob_to_qphred's log10 over (0, 1] down to subnormals and around 1 (the near-1 branch of log)."""
    lib = reflib.oracle()
    lib.ox_libm_d_mirror_check.restype = C.c_uint64
    lib.ox_libm_d_mirror_check.argtypes = [C.c_int, C.c_void_p, C.c_uint64, C.c_void_p]
    rng = np.random.default_rng(3)
    n = 2_000_000
    u = rng.random(n)
    sets = {
        0: np.concatenate([-1100.0 * u, -40.0 * rng.random(n), -rng.random(n) * rng.random(n), -745.2 + 80.0 * (rng.random(n) - 0.5), 1440.0 * (rng.random(n) - 0.5),
                           [0.0, -0.0, 1e-300, -1e-300, -708.0, -709.0, -744.0, -745.0, -745.13, -745.2, -746.0, -1023.9, -1024.0, -1e6, 709.7, 709.8, 710.0, 1024.0, -np.inf]]),
        1: np.concatenate([u, u * 1e-5, np.ldexp(u, -rng.integers(0, 1074, n).astype(np.int32)), 1.0 - 0.07 * u, 1.0 + 0.07 * u,
                           [1.0, 0.5, 1e-300, 5e-324, 1e-310, 2.2250738585072014e-308, 0.9375, 1.064697265625, 0.93749999999999989, 1.0646972656249998, 0.0]]),
        2: np.concatenate([u, np.ldexp(1.0 + u, rng.integers(-1000, 1000, n).astype(np.int32)), 0.93 + 0.14 * u, [1.0, 5e-324, 0.0]]),
        3: np.concatenate([u, 0.01 * u, np.ldexp(u, -rng.integers(0, 80, n).astype(np.int32)), -0.999999 * u, 1e6 * u, 0.41 + 0.01 * u, -0.30 + 0.02 * u, np.exp(-40.0 * u),
                           [0.0, -0.0, 1.0, 0.41421356237309503, 0.41421356237309509, -0.29289321881345243, 1e-9, 5.4e-17, 0.5, 3.0, 9007199254740994.0]]),
    }
    for kind, xs in sets.items():
        xs = np.ascontiguousarray(xs, dtype=np.float64)
        first = np.zeros(1)
        bad = lib.ox_libm_d_mirror_check(kind, xs.ctypes.data, len(xs), first.ctypes.data)
        assert bad == 0, (kind, bad, float(first[0]).hex())


def test_expf_mirror_matches_libm():
    """sx_expf (the somatic model's float log-sum: getLogSum<float> -> std::exp(float)) == glibc's expf on every 97th float bit pattern and on every
    17th float of [-104, -2^-20] (the arguments the log-sum produces); all 2^32 patterns were checked once outside the suite (0 mismatches)."""
    lib = reflib.oracle()
    lib.ox_expf_mirror_check.restype = C.c_uint64
    lib.ox_expf_mirror_check.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]
    first = np.zeros(1, np.uint32)
    assert lib.ox_expf_mirror_check(5, 0xFFFFFFFF, 97, first.ctypes.data) == 0, hex(int(first[0]))
    lo, hi = int(np.float32(-(2.0 ** -20)).view(np.uint32)), int(np.float32(-104.0).view(np.uint32))  # negative floats: bit patterns ascend with magnitude
    assert lo < hi and lib.ox_expf_mirror_check(lo, hi, 17, first.ctypes.data) == 0, hex(int(first[0]))


def test_stdsort_mirror_matches_libstdcxx():
    lib = reflib.oracle()
    rng = np.random.default_rng(2)
    for it in range(4000):
        n = int(rng.integers(0, 200)) if it % 10 else int(rng.integers(200, 3000))
        key = rng.integers(0, int(rng.integers(1, 8)), n).astype(np.uint8)
        if it % 7 == 0:
            key.sort()
        a = np.arange(n, dtype=np.uint32)
        b = np.arange(n, dtype=np.uint32)
        lib.ox_sort_restated(a.ctypes.data, n, key.ctypes.data)
        lib.ox_sort_std(b.ctypes.data, n, key.ctypes.data)
        assert np.array_equal(a, b)


def test_score_indels_oracle_against_reference_golden():
    """tests/golden/score_indels_ref.npz = the reference's own score_indels output (made by make_score_indels_golden.py)."""
    gold = np.load(os.path.join(HERE, "golden", "score_indels_ref.npz"))
    total = 0
    for case in range(specgen.SCORE_INDELS_GOLDEN_CASES):
        sb, lnp = specgen.score_indels_case(case)
        recs, n_rec, max_aln, _ = reflib.ox_score_indels(sb, lnp)
        assert np.array_equal(n_rec, gold[f"n_rec{case}"]) and np.array_equal(max_aln, gold[f"max_aln{case}"])
        assert recs.tobytes() == gold[f"recs{case}"].tobytes()
        total += len(recs)
    assert total > 200


def _k6_list_case(case):
    """A K6 batch with what score_indels_case has none of: reads without a candidate alignment (the list kernel never sees them) and
    reads with 9 to 40 alignments (the second local-memory scratch tier)."""
    rng = np.random.default_rng(7000 + case)
    regions, lnp = specgen.random_score_indels_regions(rng, 8, alns_per_read=(1, 40))
    for _win, reads in regions:
        for _ in range(int(rng.integers(1, 3))):
            reads.insert(int(rng.integers(0, len(reads) + 1)), B.ScoredReadSpec(int(rng.integers(30, 151)), [], fwd=bool(rng.random() < 0.5)))
    return B.ScoreIndelsBatch(regions), lnp


def test_k6_device_body_and_list_walk_on_the_host(tmp_path):
    """strelka_b200/csrc/k6_core.cuh is __host__ __device__: the exact per-read body the kernel runs, compiled with g++
    (tests/cpp/k6_core_host.cpp) and run on the CPU against the oracle, read by read and the way k6_score_list_kernel walks its list --
    the logic of the CUDA path is checked in the GPU-less container too.  (A test harness only: libstrelka_b200.so has no host
    execution path.)"""
    import subprocess

    root = os.path.dirname(HERE)
    so = str(tmp_path / "libk6core.so")
    subprocess.check_call(["g++", "-std=c++14", "-O2", "-fPIC", "-shared", "-I" + os.path.join(root, "include"), "-I" + os.path.join(root, "strelka_b200", "csrc"),
                           os.path.join(HERE, "cpp", "k6_core_host.cpp"), "-o", so])
    lib = C.CDLL(so)
    lib.k6core_run.argtypes = [C.POINTER(A.SxScoreIndelsBatch)] + [C.c_void_p] * 6 + [C.c_uint32, C.c_void_p]
    total = 0
    walked = np.zeros(4, np.int64)  # list walk: reads skipped (no alignment), reads per scratch tier (8/4 local, 40/4 local, arena)
    for case in range(60):
        for extra, (sb, lnp) in enumerate((specgen.score_indels_case(case), _k6_list_case(case))):
            want = reflib.ox_score_indels(sb, lnp)
            # 0: the plain per-read body; 1: what the list kernel does (sx_k6_run's memsets, then the listed reads in reverse order, each
            # with its region from k6_region_of and the scratch tier the kernel picks)
            for list_walk in (0, 1):
                out = B.ScoreIndelsOut(sb)
                for a in (out.n_rec, out.max_aln, out.eval_aln):
                    a[:] = 0xA5A5A5A5  # a read whose outputs nobody writes shows up
                st, counts = np.zeros(1, np.uint32), np.zeros(4, np.uint32)
                lib.k6core_run(C.byref(sb.c), A.ptr(lnp), A.ptr(out.recs), A.ptr(out.n_rec), A.ptr(out.max_aln), A.ptr(out.eval_aln), A.ptr(st), list_walk,
                               A.ptr(counts))
                assert st[0] == 0
                for w, g in zip(want, out.compact()):
                    assert w.tobytes() == g.tobytes()
                walked += counts
            total += 0 if extra else len(want[0])
    print("k6 list walk: skipped %d, tiers %d / %d / %d" % tuple(walked))
    assert total > 1500
    assert walked[0] > 600 and walked[1] > 1000 and walked[2] > 500 and walked[3] > 1200


def test_libm_tables_are_this_libms(tmp_path):
    """strelka_b200/csrc/sx_libm_mirror_d_tables.inc is what tools/gen_libm_d_tables.py reads out of the libm.so.6 the reference is linked against
    here (the script refuses another libm build: then the mirror tests above are the ones that matter, and this one is skipped)."""
    import shutil
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    work = tmp_path / "r"
    (work / "strelka_b200" / "csrc").mkdir(parents=True)
    shutil.copy(os.path.join(root, "tools", "gen_libm_d_tables.py"), work / "gen.py")
    r = subprocess.run([sys.executable, "gen.py"], cwd=work, capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("another libm build: " + (r.stderr or r.stdout).strip()[:200])
    assert open(work / "strelka_b200" / "csrc" / "sx_libm_mirror_d_tables.inc").read() == open(os.path.join(root, "strelka_b200", "csrc", "sx_libm_mirror_d_tables.inc")).read()


def test_bench_worker_failures_fail_the_run():
    """bench.py runs the windows of the end-to-end leg on worker threads: an exception in one of them must end the run (a worker that had died on an
    out-of-memory error once made the leg look fast in a tuning run)."""
    import importlib.util

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(root, "bench.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    done = []
    m.run_threads([lambda: done.append(1), lambda: done.append(2)])
    assert sorted(done) == [1, 2]

    def boom():
        raise RuntimeError("worker died")

    with pytest.raises(RuntimeError):
        m.run_threads([lambda: done.append(3), boom])
