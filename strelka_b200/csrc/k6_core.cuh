// k6_core.cuh -- the per-read body of K6 score_indels (include/strelka_b200.h), written once for the device.
//
// The reference keeps its per-read bookkeeping in ordered maps and sets keyed by IndelKey
// (starling_common/starling_read_align_score_indels.cpp:42-54 iks_map_t, :82 overlap_map_t, indel_set_t).  Here a read owns flat
// per-thread arrays: the evaluated indels as an ascending list of window indices, one "best score with the indel present / absent"
// pair per evaluated indel and an E x E table for the (indel, alternate indel) entries -- every map update of the reference is a
// running maximum, so the iteration order over alignments does not matter and no container is needed.
//
// The functions are __host__ __device__ so that tests/cpp/k6_core_host.cpp can single-step exactly this code on the CPU against
// the oracle (a test of the device logic; the product has no host execution path -- k6_score_indels.cu only launches the kernel).
#pragma once

#include "strelka_b200.h"

#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define K6_HD __host__ __device__ __forceinline__
#else
#define K6_HD inline
#endif

enum
{
    K6_ST_SEGKIND = 1,  // a path segment outside score_indels' domain (SKIP, REFSKIP, unknown)
    K6_ST_LIMIT_A = 2,  // more alignments than the scratch was sized for (host sizing error)
    K6_ST_LIMIT_E = 4,  // more evaluated indels than K6_MAX_EVAL
    K6_ST_RECCAP = 8,   // rec_off leaves too few output slots for a read
    K6_ST_BADKEY = 16,  // an alignment key index outside the region's window / unsupported key type
};

#define K6_MAX_EVAL 64u // evaluated indels per read (the reference has no limit; 150 bp reads see a handful)

template <class T> struct k6_strided
{
    T* p;
    size_t stride; // element i of this thread's array lives at p[i * stride] (interleaved across threads: coalesced)
    K6_HD T& operator[](const size_t i) const { return p[i * stride]; }
};

// The three kinds of maxima are kept as FLOATS: the reference keeps doubles and converts the winner to ReadPathScores::score_t
// (float) at the very end; rounding to nearest is monotone, so max_i (float)x_i == (float) max_i x_i -- same bits, half the state.
struct k6_scratch
{
    k6_strided<uint32_t> ord;   // [maxA] alignments, best score first
    k6_strided<double> smooth;  // [maxA] (compared in double against the smoothing range)
    k6_strided<uint8_t> filt;   // [maxA]
    k6_strided<uint16_t> ev;    // [maxE] evaluated window indices, ascending
    k6_strided<uint16_t> slot;  // [maxE] output slot reserved for ev[i]
    k6_strided<float> present;  // [maxE] best score, indel present   (iks key (e,(true ,e)))
    k6_strided<float> absent;   // [maxE] best score, indel absent    (iks key (e,(false,e)))
    k6_strided<uint8_t> has;    // [maxE] bit0: present set, bit1: absent set
    k6_strided<float> alt;      // [maxE*maxE] row e, column o: best score with alternate o present  (iks key (e,(true,o)))
    k6_strided<uint8_t> pair;   // [maxE*maxE] bit0: e and o conflict (orthogonalIndelMap), bit1: alt set
    uint32_t maxA, maxE;
};

// the same arrays as per-thread local memory, for reads with few alignments and few output slots (the common case: local memory is
// L1-cached write-back, the strided arena is an L2 round trip per access)
template <int MA, int ME> struct k6_local_scratch
{
    double smooth[MA];
    float present[ME], absent[ME];
    float alt[ME * ME];
    uint16_t ev[ME], slot[ME];
    uint8_t ord[MA]; // MA <= 255
    uint8_t filt[MA];
    uint8_t has[ME];
    uint8_t pair[ME * ME];
    static constexpr uint32_t maxA = MA, maxE = ME;
};

struct k6_view // device (or, in the host test, host) pointers of one batch
{
    sx_score_indels_batch b;
    const double* lnp;
    sx_read_indel_score* recs;
    uint32_t *n_rec, *max_aln, *eval_aln;
};

K6_HD bool k6_read_kind(const unsigned k) { return k == SX_SEG_MATCH || k == SX_SEG_INSERT || k == SX_SEG_SOFTCLIP; }
K6_HD bool k6_ref_kind(const unsigned k) { return k == SX_SEG_MATCH || k == SX_SEG_DELETE || k == SX_SEG_SKIP; }
K6_HD int k6_min(const int a, const int b) { return a < b ? a : b; }
K6_HD int k6_max(const int a, const int b) { return a > b ? a : b; }

// indel_util.cpp:29-45
K6_HD bool k6_conflict(const sx_indel_key& a, const sx_indel_key& b)
{
    const int64_t margin((a.type == SX_INDEL_TYPE_MISMATCH || b.type == SX_INDEL_TYPE_MISMATCH) ? 0 : 1);
    const int64_t b1(a.pos), b2(b.pos);
    return (b2 + b.del_len + margin > b1) && (b2 < b1 + a.del_len + margin);
}

struct k6_aln
{
    int32_t pos;
    const sx_aln_seg* seg;
    uint32_t n_seg;
    const uint16_t* keys;
    uint32_t n_keys;
};

K6_HD k6_aln k6_aln_at(const sx_score_indels_batch& b, const uint32_t a)
{
    k6_aln al;
    al.pos = b.aln_pos[a];
    const uint32_t s0(b.aln_seg_off[a]), k0(b.aln_key_off[a]);
    al.seg = b.segs + s0;
    al.n_seg = b.aln_seg_off[a + 1] - s0;
    al.keys = b.aln_keys + k0;
    al.n_keys = b.aln_key_off[a + 1] - k0;
    return al;
}

K6_HD bool k6_contains(const k6_aln& al, const uint32_t key)
{
    for (uint32_t i = 0; i < al.n_keys; ++i)
        if (al.keys[i] == key) return true;
    return false;
}

// starling_read_align.cpp:1280-1320
struct k6_path_stats
{
    unsigned indelCount, totalDeletionSize, totalInsertionSize, sumSegmentPos;
};

K6_HD k6_path_stats k6_stats_of(const k6_aln& al)
{
    k6_path_stats e = {0, 0, 0, 0};
    unsigned read_pos(0);
    for (uint32_t s = 0; s < al.n_seg; ++s)
    {
        const unsigned kind(al.seg[s].kind), len(al.seg[s].len);
        if (kind != SX_SEG_MATCH) e.indelCount++;
        if (kind == SX_SEG_DELETE)
        {
            e.totalDeletionSize += len;
            e.sumSegmentPos += read_pos;
        }
        if (kind == SX_SEG_INSERT)
        {
            e.totalInsertionSize += len;
            e.sumSegmentPos += read_pos;
        }
        if (k6_read_kind(kind)) read_pos += len;
    }
    return e;
}

K6_HD unsigned k6_candidate_count(const sx_indel_key* win, const k6_aln& al)
{
    unsigned n(0);
    for (uint32_t i = 0; i < al.n_keys; ++i) n += (win[al.keys[i]].flags & SX_IKF_CANDIDATE) ? 1u : 0u;
    return n;
}

// isFirstCandidateAlignmentPreferred, starling_read_align.cpp:1352-1377
K6_HD bool k6_first_preferred(const sx_indel_key* win, const k6_aln& c1, const k6_aln& c2)
{
    const k6_path_stats e1(k6_stats_of(c1)), e2(k6_stats_of(c2));
    if (e2.indelCount != e1.indelCount) return e2.indelCount > e1.indelCount;
    const unsigned cic1(k6_candidate_count(win, c1)), cic2(k6_candidate_count(win, c2));
    if (cic2 != cic1) return cic2 < cic1;
    if (e2.totalInsertionSize != e1.totalInsertionSize) return e2.totalInsertionSize > e1.totalInsertionSize;
    if (e2.totalDeletionSize != e1.totalDeletionSize) return e2.totalDeletionSize > e1.totalDeletionSize;
    return e2.sumSegmentPos >= e1.sumSegmentPos;
}

// get_alignment_indel_bp_overlap, score_indels.cpp:131-234: max(left, right) overlap, or -1 for a segment kind it asserts on
K6_HD int k6_bp_overlap(const int oligo, const k6_aln& al, const bool fwd, const sx_indel_key& ik)
{
    int32_t read_head(0), ref_head(al.pos);
    bool is_left(false), is_right(false);
    int32_t left_read(0), right_read(0);
    const int32_t ik_right(ik.pos + (int32_t)ik.del_len);
    for (uint32_t s = 0; s < al.n_seg; ++s)
    {
        const unsigned kind(al.seg[s].kind);
        const int32_t len(al.seg[s].len);
        int32_t next_read(read_head), next_ref(ref_head);
        if (kind == SX_SEG_MATCH)
        {
            next_read += len;
            next_ref += len;
        }
        else if (kind == SX_SEG_INSERT) next_read += len;
        else if (kind == SX_SEG_DELETE) next_ref += len;
        else if (kind != SX_SEG_SOFTCLIP && kind != SX_SEG_HARDCLIP) return -1;
        if (!is_left && ik.pos <= next_ref)
        {
            left_read = read_head + (ik.pos - ref_head);
            is_left = true;
        }
        if (!is_right && ik_right < next_ref)
        {
            right_read = read_head + (ik_right - ref_head);
            is_right = true;
        }
        read_head = next_read;
        ref_head = next_ref;
    }
    int left_ext(0), right_ext(0);
    if (fwd)
    {
        if (left_read > 0) left_ext = oligo;
    }
    else if ((read_head - right_read) > 0) right_ext = oligo;
    int left(0), right(0);
    if (is_left) left = k6_max(0, k6_min(left_read + left_ext, read_head - left_read));
    if (is_right) right = k6_max(0, k6_min(right_read, (read_head - right_read) + right_ext));
    return k6_max(left, right);
}

// get_soft_clip_alignment_range, alignment_util.cpp:45-55
K6_HD void k6_soft_clip_range(const k6_aln& al, int32_t& begin, int32_t& end)
{
    int32_t lead(0), trail(0), asize(0);
    bool in_lead(true);
    for (uint32_t s = 0; s < al.n_seg; ++s)
    {
        const unsigned kind(al.seg[s].kind);
        const int32_t len(al.seg[s].len);
        if (k6_ref_kind(kind)) asize += len;
        if (kind == SX_SEG_HARDCLIP || kind == SX_SEG_SOFTCLIP) continue;
        if (kind == SX_SEG_INSERT)
        {
            if (in_lead) lead += len;
            trail += len; // an insertion run that is still unbroken at the end of the path is the trailing one
        }
        else
        {
            in_lead = false;
            trail = 0;
        }
    }
    begin = al.pos - lead;
    end = al.pos + asize + trail;
}

// getLowestFwdReadPosForRefRange, alignment_util.cpp:222-302
K6_HD int32_t k6_lowest_fwd_read_pos(const k6_aln& al, const bool fwd, const int32_t range_begin, const int32_t range_end)
{
    const int32_t target((fwd ? range_begin : range_end - 1) - al.pos);
    if (target < 0) return -1;
    int32_t ref_offset(0), read_offset(0), readOffset(-1), readLength(0);
    bool done(false);
    for (uint32_t s = 0; s < al.n_seg; ++s)
    {
        const unsigned kind(al.seg[s].kind);
        const int32_t len(al.seg[s].len);
        const bool rk(k6_read_kind(kind));
        if (rk) readLength += len;
        if (done) continue;
        if (rk) read_offset += len;
        if (!k6_ref_kind(kind)) continue;
        ref_offset += len;
        if (ref_offset <= target) continue;
        done = true;
        if (rk) readOffset = read_offset - (ref_offset - target);
    }
    if (readOffset < 0) return -1;
    return fwd ? readOffset : readLength - (readOffset + 1);
}

K6_HD void k6_tick(float& slot, uint8_t& flags, const uint8_t bit, const double lnp)
{
    const float f((float)lnp); // see k6_scratch: the maximum of the rounded values is the rounded maximum
    if ((flags & bit) && slot >= f) return; // updateIndelScoringInfo, score_indels.cpp:60-75
    slot = f;
    flags |= bit;
}

/// everything score_indels does for read r of `region`; returns K6_ST_* bits (0 = fine).  SC: k6_scratch or k6_local_scratch.
template <class SC> K6_HD uint32_t k6_score_read(const k6_view& v, const uint32_t region, const uint32_t r, SC& S)
{
    const sx_score_indels_batch& b(v.b);
    const sx_score_indels_opts& opt(b.opts);
    const sx_indel_key* win(b.keys + b.region_key_off[region]);
    const uint32_t n_win(b.region_key_off[region + 1] - b.region_key_off[region]);
    const uint32_t a0(b.aln_off[r]), n_cal(b.aln_off[r + 1] - a0);
    v.n_rec[r] = 0;
    v.max_aln[r] = v.eval_aln[r] = UINT32_MAX;
    if (n_cal == 0) return 0;
    if (n_cal > S.maxA) return K6_ST_LIMIT_A;
    const unsigned rflags(b.read_flags[r]);
    const bool fwd(rflags & SX_SIF_FWD);
    const double* score(v.lnp + a0);

    // ---- validation the reference leaves to its containers / asserts
    for (uint32_t c = 0; c < n_cal; ++c)
    {
        const k6_aln al(k6_aln_at(b, a0 + c));
        for (uint32_t s = 0; s < al.n_seg; ++s)
        {
            const unsigned kind(al.seg[s].kind);
            if (kind == SX_SEG_REFSKIP || kind >= SX_SEG_SKIP) return K6_ST_SEGKIND;
        }
        for (uint32_t i = 0; i < al.n_keys; ++i)
            if (al.keys[i] >= n_win) return K6_ST_BADKEY;
    }

    // ---- scoreCandidateAlignments' arg-max, starling_read_align.cpp:1573-1593
    double maxScore(score[0]);
    uint32_t maxCal(0);
    for (uint32_t c = 1; c < n_cal; ++c)
    {
        const double path_lnp(score[c]);
        if (path_lnp < maxScore) continue;
        if ((path_lnp <= maxScore) && k6_first_preferred(win, k6_aln_at(b, a0 + maxCal), k6_aln_at(b, a0 + c))) continue;
        maxScore = path_lnp;
        maxCal = c;
    }
    v.max_aln[r] = a0 + maxCal;

    // ---- late_indel_normalization_filter, score_indels.cpp:281-450 (its nonnorm_indels is a by-value argument: only the filter
    // flags and the re-chosen maximum leave the function)
    {
        const double equiv_range(opt.is_smoothed_alignments ? opt.smoothed_lnp_range : 0.);
        // std::sort(rbegin, rend) of (score, index) pairs == descending lexicographic order; insertion sort (n_cal is small)
        for (uint32_t c = 0; c < n_cal; ++c)
        {
            S.smooth[c] = score[c];
            S.filt[c] = 0;
            uint32_t j(c);
            for (; j > 0; --j)
            {
                const uint32_t p(S.ord[j - 1]);
                if (score[p] > score[c] || (score[p] == score[c] && p > c)) break;
                S.ord[j] = p;
            }
            S.ord[j] = c;
        }
        bool any_excluded(false);
        for (uint32_t i1 = 0; i1 < n_cal; ++i1)
        {
            const uint32_t s1(S.ord[i1]);
            if (S.filt[s1]) continue;
            const k6_aln c1(k6_aln_at(b, a0 + s1));
            for (uint32_t i2 = i1 + 1; i2 < n_cal; ++i2)
            {
                const uint32_t s2(S.ord[i2]);
                if (S.filt[s2]) continue;
                if (S.smooth[s2] + equiv_range < S.smooth[s1]) break;
                // is_equiv_candidate, :247-276; only the first differing pair decides which alignment goes
                const k6_aln c2(k6_aln_at(b, a0 + s2));
                if (c1.n_keys != c2.n_keys) continue;
                bool equiv(true), have_pair(false);
                uint32_t p1(0), p2(0);
                for (uint32_t i = 0; i < c1.n_keys; ++i)
                {
                    const uint32_t k1(c1.keys[i]), k2(c2.keys[i]);
                    if (k1 == k2) continue;
                    const sx_indel_key &x(win[k1]), &y(win[k2]);
                    if (x.type != y.type || x.del_len != y.del_len || x.ins_len != y.ins_len || x.ins_id != y.ins_id)
                    {
                        equiv = false;
                        break;
                    }
                    if (!have_pair)
                    {
                        have_pair = true;
                        p1 = k1;
                        p2 = k2;
                    }
                }
                if (!equiv || !have_pair) continue;
                // is_first_indel_dominant, :285-300
                const bool ic1(win[p1].flags & SX_IKF_CANDIDATE), ic2(win[p2].flags & SX_IKF_CANDIDATE);
                const bool first_dominant((ic2 && !ic1) ? false : (ic2 == ic1) ? (win[p1].pos <= win[p2].pos) : true);
                any_excluded = true;
                const double sm(S.smooth[s1] > S.smooth[s2] ? S.smooth[s1] : S.smooth[s2]);
                if (first_dominant)
                {
                    S.filt[s2] = 1;
                    S.smooth[s1] = sm;
                }
                else
                {
                    S.filt[s1] = 1;
                    S.smooth[s2] = sm;
                    break;
                }
            }
        }
        if (any_excluded)
            for (uint32_t i = 0; i < n_cal; ++i)
            {
                const uint32_t s(S.ord[i]);
                if (S.filt[s]) continue;
                maxScore = score[s];
                maxCal = s;
                break;
            }
    }
    v.eval_aln[r] = a0 + maxCal;
    const k6_aln maxAl(k6_aln_at(b, a0 + maxCal));

    sx_read_indel_score* out(v.recs + b.rec_off[r]);
    const uint32_t out_cap(b.rec_off[r + 1] - b.rec_off[r]);
    uint32_t n_out(0), E(0);

    // ---- (2a) which indels this read evaluates, :520-656.  Records are reserved in key order: a suboverlap mark is final, an
    // evaluated indel gets a placeholder (flags 0) that step (3) fills or leaves dead.
    {
        int32_t rb, re;
        k6_soft_clip_range(maxAl, rb, re);
        // IndelBuffer::rangeIterator(rb, re), IndelBuffer.cpp:76-91
        uint32_t k(0);
        while (k < n_win && (int64_t)win[k].pos < (int64_t)rb - (int64_t)opt.max_indel_size) k++;
        for (; k < n_win && win[k].pos < re; ++k)
            if (win[k].pos + (int32_t)win[k].del_len >= rb) break;
        for (; k < n_win && win[k].pos < re; ++k)
        {
            const sx_indel_key ik(win[k]);
            if (ik.type == SX_INDEL_TYPE_MISMATCH) continue;
            if (ik.type != SX_INDEL_TYPE_INDEL) return K6_ST_BADKEY;
            if (!(ik.flags & SX_IKF_CANDIDATE)) continue;
            int best(-1);
            if (k6_contains(maxAl, k)) best = (int)maxCal;
            else
            {
                double bestScore(0);
                for (uint32_t c = 0; c < n_cal; ++c)
                {
                    if (c == maxCal || S.filt[c]) continue;
                    if (!k6_contains(k6_aln_at(b, a0 + c), k)) continue;
                    if (best < 0 || score[c] > bestScore)
                    {
                        bestScore = score[c];
                        best = (int)c;
                    }
                }
            }
            if (best < 0) continue;
            const int bpo(k6_bp_overlap((int)opt.upstream_oligo_size, k6_aln_at(b, a0 + best), fwd, ik));
            const bool sub(bpo < opt.min_read_bp_flank);
            if (sub && bpo <= 0) continue;
            if (n_out >= out_cap) return K6_ST_RECCAP;
            sx_read_indel_score rec = {};
            rec.key = (uint16_t)k;
            rec.flags = sub ? SX_RIS_SUBOVERLAP : 0;
            out[n_out] = rec;
            if (!sub)
            {
                if (E >= S.maxE) return K6_ST_LIMIT_E;
                S.ev[E] = (uint16_t)k;
                S.slot[E] = (uint16_t)n_out;
                S.has[E] = 0;
                ++E;
            }
            ++n_out;
        }
    }

    // ---- orthogonalIndelMap, :665-686
    for (uint32_t i = 0; i < E; ++i)
        for (uint32_t j = 0; j < E; ++j) S.pair[i * S.maxE + j] = (i != j && k6_conflict(win[S.ev[i]], win[S.ev[j]])) ? 1 : 0;

    // ---- (2b) best score of every (indel, state), :688-849
    for (uint32_t c = 0; c < n_cal; ++c)
    {
        if (S.filt[c]) continue;
        const double sc(score[c]);
        const k6_aln al(k6_aln_at(b, a0 + c));
        for (uint32_t ei = 0; ei < E; ++ei)
        {
            const uint32_t e(S.ev[ei]);
            const sx_indel_key ek(win[e]);
            if (k6_contains(al, e))
            {
                k6_tick(S.present[ei], S.has[ei], 1, sc);
                const double asRefError(sc + ek.ref_to_indel_lnp);
                k6_tick(S.absent[ei], S.has[ei], 2, asRefError);
                for (uint32_t oj = 0; oj < E; ++oj)
                {
                    if (!(S.pair[ei * S.maxE + oj] & 1)) continue;
                    k6_tick(S.absent[oj], S.has[oj], 2, asRefError);
                    k6_tick(S.alt[oj * S.maxE + ei], S.pair[oj * S.maxE + ei], 2, sc);
                }
            }
            else
            {
                // which_interfering_indel, :100-118
                int interfering(-1);
                for (uint32_t i = 0; i < al.n_keys; ++i)
                {
                    const sx_indel_key& cur(win[al.keys[i]]);
                    if (cur.type == SX_INDEL_TYPE_MISMATCH) continue;
                    if (k6_conflict(cur, ek))
                    {
                        interfering = (int)al.keys[i];
                        break;
                    }
                }
                k6_tick(S.present[ei], S.has[ei], 1, sc + ek.indel_to_ref_lnp);
                if (interfering < 0) k6_tick(S.absent[ei], S.has[ei], 2, sc);
                else
                {
                    bool evaluated(false);
                    for (uint32_t j = 0; j < E; ++j) evaluated |= (S.ev[j] == (uint32_t)interfering);
                    if (!evaluated)
                    {
                        // nonCandidateIndelsOrthogonalToEvaluationIndels, :816-845 (a maximum: repeats are harmless)
                        const sx_indel_key nc(win[interfering]);
                        for (uint32_t j = 0; j < E; ++j)
                            if (k6_conflict(nc, win[S.ev[j]])) k6_tick(S.absent[j], S.has[j], 2, sc + nc.ref_to_indel_lnp);
                    }
                }
            }
        }
    }

    // ---- (3) one ReadPathScores per evaluated indel, :852-1075
    const unsigned read_length(b.read_len[r]);
    const unsigned fullReadLength(b.full_len ? b.full_len[r] : read_length);
    const unsigned fullReadOffset(b.full_off ? b.full_off[r] : 0);
    uint32_t n_dead(0);
    for (uint32_t ei = 0; ei < E; ++ei)
    {
        const uint32_t e(S.ev[ei]);
        float indelScore((float)maxScore);
        if (!k6_contains(maxAl, e))
        {
            if (!(S.has[ei] & 1))
            {
                ++n_dead;
                continue;
            }
            indelScore = S.present[ei];
        }
        if (!(S.has[ei] & 2))
        {
            ++n_dead;
            continue;
        }
        const float refScore(S.absent[ei]);
        const sx_indel_key ek(win[e]);
        const int32_t right_pos(ek.pos + (int32_t)ek.del_len);
        const int32_t readPos(k6_lowest_fwd_read_pos(maxAl, fwd, ek.pos - 1, right_pos + 1));
        const int32_t revReadPos(k6_lowest_fwd_read_pos(maxAl, !fwd, ek.pos - 1, right_pos + 1));
        int32_t dist((int32_t)fullReadLength);
        if (readPos >= 0) dist = readPos + (int32_t)fullReadOffset;
        if (revReadPos >= 0)
        {
            const int32_t fullRev((int32_t)((uint32_t)revReadPos + (fullReadLength - (fullReadOffset + read_length))));
            if (fullRev < dist) dist = fullRev;
        }
        sx_read_indel_score rec = {};
        rec.key = (uint16_t)e;
        rec.flags = SX_RIS_SCORED;
        rec.ref_lnp = refScore;
        rec.indel_lnp = indelScore;
        rec.read_pos = (int16_t)readPos;
        rec.dist_from_edge = (int16_t)dist;
        // ReadPathScores::insertAlt, IndelData.cpp:42-68, over orthogonalIndelMap[e] in key order
        unsigned n_alt(0);
        for (uint32_t oj = 0; oj < E; ++oj)
        {
            const unsigned pr(S.pair[ei * S.maxE + oj]);
            if ((pr & 3) != 3) continue;
            const float a(S.alt[ei * S.maxE + oj]);
            if (n_alt < 2)
            {
                rec.alt_key[n_alt] = S.ev[oj];
                rec.alt_lnp[n_alt] = a;
                ++n_alt;
            }
            else
            {
                unsigned min_index(2);
                float mn(a);
                for (unsigned i = 0; i < 2; ++i)
                    if (rec.alt_lnp[i] < mn)
                    {
                        mn = rec.alt_lnp[i];
                        min_index = i;
                    }
                if (min_index < 2)
                {
                    rec.alt_key[min_index] = S.ev[oj];
                    rec.alt_lnp[min_index] = a;
                }
            }
        }
        rec.n_alt = (uint8_t)n_alt;
        out[S.slot[ei]] = rec;
    }
    // drop the placeholders step (3) skipped (rare: an indel no surviving alignment carries, or none without it)
    uint32_t w(n_out);
    if (n_dead)
    {
        w = 0;
        for (uint32_t i = 0; i < n_out; ++i)
        {
            if (out[i].flags == 0) continue;
            if (w != i) out[w] = out[i];
            ++w;
        }
    }
    v.n_rec[r] = w;
    return 0;
}

/// the region of read r: the last region whose first read is <= r (the reads of a region are consecutive)
K6_HD uint32_t k6_region_of(const uint32_t* region_read_off, const uint32_t n_regions, const uint32_t r)
{
    uint32_t lo(0), hi(n_regions);
    while (hi - lo > 1)
    {
        const uint32_t mid((lo + hi) >> 1);
        if (region_read_off[mid] <= r) lo = mid;
        else hi = mid;
    }
    return lo;
}

#define K6_FAST_A 8
#define K6_FAST_E 4
#define K6_MID_A 40 /* second local-memory tier: a profile put a large share of the kernel's instructions on the strided-arena accessor once most reads had > 8 alignments */

/// which scratch the body of read r runs with: 0 = k6_local_scratch<K6_FAST_A, K6_FAST_E>, 1 = k6_local_scratch<K6_MID_A, K6_FAST_E>, 2 = the arena
K6_HD unsigned k6_scratch_tier(const sx_score_indels_batch& b, const uint32_t r)
{
    const uint32_t n_cal(b.aln_off[r + 1] - b.aln_off[r]), slots(b.rec_off[r + 1] - b.rec_off[r]);
    if (n_cal <= K6_FAST_A && slots <= K6_FAST_E) return 0;
    if (n_cal <= K6_MID_A && slots <= K6_FAST_E) return 1; // (whole-path windows: 12 candidate alignments per realigned read on average, a few dozen at most)
    return 2;
}

/// read r of `region` with the cheapest scratch that fits (k6_scratch_tier); S is the arena, for reads too deep for local memory
K6_HD uint32_t k6_score_read_tiered(const k6_view& v, const uint32_t region, const uint32_t r, k6_scratch& S)
{
    const unsigned tier(k6_scratch_tier(v.b, r));
    if (tier == 0)
    {
        k6_local_scratch<K6_FAST_A, K6_FAST_E> L;
        return k6_score_read(v, region, r, L);
    }
    if (tier == 1)
    {
        k6_local_scratch<K6_MID_A, K6_FAST_E> L;
        return k6_score_read(v, region, r, L);
    }
    return k6_score_read(v, region, r, S);
}
