// k9_core.cuh -- the per-read body of K9 choose_realignment (include/strelka_b200.h): from a read's candidate alignments and their
// scores to rseg.realignment.  Restates the tail of scoreCandidateAlignments (starling_common/starling_read_align.cpp:1573-1741, unpinned
// reads, isTestSoftClippedInputAligned = false), isFirstCandidateAlignmentPreferred :1352-1377, finishRealignment :1411-1450 and
// starling_read_align_clipper.cpp (get_alignment_ref_map :96-146, mark_ref_map_conflicts :150-225, soft_clip_alignment :255-338,
// getClippedAlignmentFromTopAlignmentPool :340-424).  The pool is never stored: membership is a comparison, so the alignments are
// simply walked again, and so is the reference map: it is piecewise (one type per segment, a MATCH position that is the segment's start
// plus the read offset), so a member conflicts with it on whole segment overlaps, and the clip walk needs only the 32-position words at the
// ends that hold the first and the last unconflicted match.  __host__ __device__: tests/cpp/k9_core_host.cpp runs exactly this code on the
// CPU against the reference.
#pragma once

#include "strelka_b200.h"

#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define K9_HD __host__ __device__ __forceinline__
#else
#define K9_HD inline
#endif

#define K9_MAX_READ 1024u // read positions of the reference map (longer: SX_REALIGN_ST_LIMIT)

enum // ref_map_type::map_t, starling_read_align_clipper.cpp:44-51
{
    K9_NONE = 0,
    K9_MATCH = 1,
    K9_INSERT = 2,
    K9_SOFT_CLIP = 3,
    K9_CONFLICT = 4
};

struct k9_view
{
    sx_realign_batch b;
    const double* lnp;
};

struct k9_scratch // per thread (no longer read: the map is not stored)
{
    uint8_t* type; // [K9_MAX_READ]
    int32_t* pos;  // [K9_MAX_READ]
};

K9_HD bool k9_align_match(const unsigned t) { return t == SX_AP_MATCH || t == SX_AP_SEQ_MATCH || t == SX_AP_SEQ_MISMATCH; }
K9_HD bool k9_read_len_kind(const unsigned t) { return t == SX_AP_MATCH || t == SX_AP_INSERT || t == SX_AP_SOFT_CLIP || t == SX_AP_SEQ_MATCH || t == SX_AP_SEQ_MISMATCH; }

struct k9_epi // extra_path_info, :1280-1291
{
    unsigned indelCount, totalDeletionSize, totalInsertionSize, sumSegmentPos, candidates;
};

K9_HD k9_epi k9_epi_of(const k9_view& v, const uint32_t k0, const uint32_t a) // getExtraPathInfo :1293-1318 + getCandidateIndelCount :1322-1334
{
    k9_epi e = {0, 0, 0, 0, 0};
    unsigned read_pos(0);
    for (uint32_t s = v.b.aln_seg_off[a]; s < v.b.aln_seg_off[a + 1]; ++s)
    {
        const unsigned t(v.b.segs[s].kind), len(v.b.segs[s].len);
        if (!k9_align_match(t)) e.indelCount++;
        if (t == SX_AP_DELETE)
        {
            e.totalDeletionSize += len;
            e.sumSegmentPos += read_pos;
        }
        if (t == SX_AP_INSERT)
        {
            e.totalInsertionSize += len;
            e.sumSegmentPos += read_pos;
        }
        if (k9_read_len_kind(t)) read_pos += len;
    }
    for (uint32_t q = v.b.aln_key_off[a]; q < v.b.aln_key_off[a + 1]; ++q) e.candidates += (v.b.keys[k0 + v.b.aln_keys[q]].flags & SX_IKF_CANDIDATE) ? 1u : 0u;
    return e;
}

K9_HD bool k9_first_preferred(const k9_epi& e1, const k9_epi& e2) // :1352-1377
{
    if (e2.indelCount != e1.indelCount) return e2.indelCount > e1.indelCount;
    if (e2.candidates != e1.candidates) return e2.candidates < e1.candidates;
    if (e2.totalInsertionSize != e1.totalInsertionSize) return e2.totalInsertionSize > e1.totalInsertionSize;
    if (e2.totalDeletionSize != e1.totalDeletionSize) return e2.totalDeletionSize > e1.totalDeletionSize;
    return e2.sumSegmentPos >= e1.sumSegmentPos;
}

// the slots a read's realignment may need: its longest candidate path + a leading and a trailing soft clip
K9_HD uint32_t k9_slots(const sx_realign_batch& b, const uint32_t r)
{
    uint32_t m(0);
    for (uint32_t a = b.aln_off[r]; a < b.aln_off[r + 1]; ++a)
    {
        const uint32_t n(b.aln_seg_off[a + 1] - b.aln_seg_off[a]);
        m = n > m ? n : m;
    }
    m = m ? m + 2 : 0;
    if (b.raw_seg_off)
    {
        const uint32_t nr(b.raw_seg_off[r + 1] - b.raw_seg_off[r]);
        m = nr > m ? nr : m;
    }
    return m;
}

K9_HD uint8_t k9_out_kind(const sx_realign_batch& b, const unsigned t)
{
    if (!b.k4_kinds) return (uint8_t)t;
    switch (t)
    {
    case SX_AP_MATCH:
    case SX_AP_SEQ_MATCH:
    case SX_AP_SEQ_MISMATCH: return SX_SEG_MATCH;
    case SX_AP_INSERT: return SX_SEG_INSERT;
    case SX_AP_DELETE: return SX_SEG_DELETE;
    case SX_AP_SKIP: return SX_SEG_SKIP;
    case SX_AP_SOFT_CLIP: return SX_SEG_SOFTCLIP;
    default: return SX_SEG_HARDCLIP;
    }
}

struct k9_writer // new_al of soft_clip_alignment: segments appended to the read's slots
{
    sx_aln_seg* out;
    uint32_t n, cap;
    bool ok;
};
K9_HD void k9_push(k9_writer& w, const unsigned type, const uint32_t len)
{
    if (w.n >= w.cap)
    {
        w.ok = false;
        return;
    }
    w.out[w.n].kind = (uint8_t)type;
    w.out[w.n].len = (uint16_t)len;
    w.out[w.n].flags = 0;
    w.n++;
}
K9_HD void k9_extend_or_add_sc(k9_writer& w, const uint32_t len) // :229-243
{
    if (w.n > 0 && w.out[w.n - 1].kind == SX_AP_SOFT_CLIP) w.out[w.n - 1].len = (uint16_t)(w.out[w.n - 1].len + len);
    else k9_push(w, SX_AP_SOFT_CLIP, len);
}

K9_HD uint32_t k9_ctz(const uint32_t x)
{
#if defined(__CUDA_ARCH__)
    return (uint32_t)(__ffs(x) - 1);
#else
    return (uint32_t)__builtin_ctz(x);
#endif
}
K9_HD uint32_t k9_clz(const uint32_t x)
{
#if defined(__CUDA_ARCH__)
    return (uint32_t)__clz(x);
#else
    return (uint32_t)__builtin_clz(x);
#endif
}

// the next segment of a path that covers read positions (ref_map_type of get_alignment_ref_map): [rb, re), its type and, for a MATCH, its
// reference position minus its read position
struct k9_cursor
{
    const sx_aln_seg* p;
    uint32_t s, n, rb, re;
    int32_t ref, off;
    uint8_t type;
};
K9_HD bool k9_next(k9_cursor& c)
{
    c.rb = c.re;
    for (; c.s < c.n; ++c.s)
    {
        const unsigned t(c.p[c.s].kind), len(c.p[c.s].len);
        if (k9_align_match(t) || t == SX_AP_INSERT || t == SX_AP_SOFT_CLIP)
        {
            c.re = c.rb + len;
            c.type = k9_align_match(t) ? K9_MATCH : (t == SX_AP_INSERT ? K9_INSERT : K9_SOFT_CLIP);
            c.off = c.ref - (int32_t)c.rb;
            if (k9_align_match(t)) c.ref += (int32_t)len;
            ++c.s;
            return true;
        }
        if (t == SX_AP_DELETE || t == SX_AP_SKIP) c.ref += (int32_t)len;
    }
    return false;
}
K9_HD k9_cursor k9_cursor_of(const k9_view& v, const uint32_t a)
{
    k9_cursor c;
    c.p = v.b.segs + v.b.aln_seg_off[a];
    c.s = 0;
    c.n = v.b.aln_seg_off[a + 1] - v.b.aln_seg_off[a];
    c.rb = c.re = 0;
    c.ref = v.b.aln_pos[a];
    c.off = 0;
    c.type = K9_NONE;
    return c;
}
// bits of [x, y) in the word of read positions w0 .. w0 + 31
K9_HD uint32_t k9_bits(const uint32_t x, const uint32_t y, const uint32_t w0)
{
    const uint32_t lo(x > w0 ? x - w0 : 0u), hi(y - w0 < 32u ? y - w0 : 32u);
    if (y <= w0 || lo >= hi) return 0u;
    return (hi == 32u ? 0xFFFFFFFFu : ((1u << hi) - 1u)) & ~((1u << lo) - 1u);
}

// read positions w0 .. w0 + 31 of the chosen alignment's reference map after mark_ref_map_conflicts (:150-225): its MATCH and SOFT_CLIP
// positions, and the positions where a member of the pool disagrees with it (another type, or a MATCH at another reference position)
K9_HD void k9_word(const k9_view& v, const uint32_t a0, const uint32_t a1, const uint32_t best, const double range, const double maxScore, const uint32_t w0,
                   uint32_t& match, uint32_t& soft, uint32_t& conflict)
{
    match = soft = conflict = 0;
    const uint32_t w1(w0 + 32u);
    k9_cursor c(k9_cursor_of(v, best));
    while (k9_next(c) && c.rb < w1)
    {
        if (c.type == K9_MATCH) match |= k9_bits(c.rb, c.re, w0);
        else if (c.type == K9_SOFT_CLIP) soft |= k9_bits(c.rb, c.re, w0);
    }
    for (uint32_t a = a0; a < a1; ++a)
    {
        if (a == best || v.lnp[a] + range < maxScore) continue;
        k9_cursor m(k9_cursor_of(v, a)), c2(k9_cursor_of(v, best));
        bool have(k9_next(c2));
        while (k9_next(m) && m.rb < w1)
        {
            if (m.re <= w0) continue;
            const uint32_t lo(m.rb > w0 ? m.rb : w0), hi(m.re < w1 ? m.re : w1);
            while (have && c2.re <= lo) have = k9_next(c2);
            while (have && c2.rb < hi)
            {
                if (c2.type != m.type || (m.type == K9_MATCH && c2.off != m.off)) conflict |= k9_bits(lo > c2.rb ? lo : c2.rb, hi < c2.re ? hi : c2.re, w0);
                if (c2.re > hi) break;
                have = k9_next(c2);
            }
        }
    }
}

// one read.  slots: where its realignment goes (cap of them).  Returns the status byte.
K9_HD uint32_t k9_read(const k9_view& v, const uint32_t region, const uint32_t r, k9_scratch& S, sx_aln_seg* slots, const uint32_t cap, int32_t& out_pos, uint16_t& out_n,
                       uint32_t& best_aln)
{
    const sx_realign_batch& b(v.b);
    const uint32_t a0(b.aln_off[r]), a1(b.aln_off[r + 1]), k0(b.region_key_off[region]);
    out_pos = 0;
    out_n = 0;
    best_aln = UINT32_MAX;
    if (a0 == a1) return 0;
    if (b.pin_flags && b.pin_flags[r]) return SX_REALIGN_ST_UNSUPPORTED;
    // ---- the maximum, :1573-1593
    double maxScore(0);
    k9_epi maxEpi = {0, 0, 0, 0, 0};
    bool have(false);
    for (uint32_t a = a0; a < a1; ++a)
    {
        const double s(v.lnp[a]);
        if (have)
        {
            if (s < maxScore) continue;
            if (s <= maxScore && k9_first_preferred(maxEpi, k9_epi_of(v, k0, a))) continue;
        }
        maxScore = s;
        maxEpi = k9_epi_of(v, k0, a);
        have = true;
    }
    // ---- the smooth pool and its preferred member, :1659-1683 (unpinned: max_allowed_path_lnp is the maximum)
    const double range(b.is_smoothed_alignments ? b.smoothed_lnp_range : 0.);
    uint32_t best(UINT32_MAX), poolSize(0);
    k9_epi bestEpi = {0, 0, 0, 0, 0};
    for (uint32_t a = a0; a < a1; ++a)
    {
        if (v.lnp[a] + range < maxScore) continue;
        ++poolSize;
        const k9_epi e(k9_epi_of(v, k0, a));
        if (best == UINT32_MAX || !k9_first_preferred(bestEpi, e))
        {
            best = a;
            bestEpi = e;
        }
    }
    if (best == UINT32_MAX) return SX_REALIGN_ST_BADPATH; // assert :1685
    best_aln = best;
    const sx_aln_seg* path(b.segs + b.aln_seg_off[best]);
    const uint32_t n_path(b.aln_seg_off[best + 1] - b.aln_seg_off[best]);
    uint32_t lead_clip(0), trail_clip(0), read_size(0);
    bool clip(false);
    if (poolSize > 1)
    {
        // ---- get_alignment_ref_map of the chosen alignment: its read length, and the statuses of the walk
        for (uint32_t s = 0; s < n_path; ++s)
        {
            const unsigned t(path[s].kind), len(path[s].len);
            if (k9_align_match(t) || t == SX_AP_INSERT || t == SX_AP_SOFT_CLIP)
            {
                if (read_size + len > K9_MAX_READ) return SX_REALIGN_ST_LIMIT;
                read_size += len;
            }
            else if (!(t == SX_AP_DELETE || t == SX_AP_SKIP || t == SX_AP_HARD_CLIP)) return SX_REALIGN_ST_BADPATH;
        }
        // ---- the statuses of mark_ref_map_conflicts for every other member of the pool
        for (uint32_t a = a0; a < a1; ++a)
        {
            if (a == best || v.lnp[a] + range < maxScore) continue;
            uint32_t read_head(0);
            for (uint32_t s = b.aln_seg_off[a]; s < b.aln_seg_off[a + 1]; ++s)
            {
                const unsigned t(b.segs[s].kind), len(b.segs[s].len);
                if (k9_align_match(t) || t == SX_AP_INSERT || t == SX_AP_SOFT_CLIP)
                {
                    if (read_head + len > read_size) return SX_REALIGN_ST_BADPATH; // the reference would index past its vector
                    read_head += len;
                }
                else if (!(t == SX_AP_DELETE || t == SX_AP_SKIP || t == SX_AP_HARD_CLIP)) return SX_REALIGN_ST_BADPATH;
            }
        }
        // ---- from each end: in until a match, then out until a conflict or a soft clip, :384-409.  Word by word from each end: lead_clip is one
        // past the last conflict / soft clip before the first unconflicted match, trail_clip the first one after the last (none: 0 / read_size)
        const uint32_t n_words((read_size + 31u) / 32u);
        for (uint32_t w = 0; w < n_words; ++w)
        {
            uint32_t m, sc, cf;
            k9_word(v, a0, a1, best, range, maxScore, 32u * w, m, sc, cf);
            const uint32_t valid(read_size - 32u * w >= 32u ? 0xFFFFFFFFu : (1u << (read_size - 32u * w)) - 1u);
            const uint32_t free_match(m & ~cf & valid), stop((cf | sc) & valid);
            if (free_match)
            {
                const uint32_t below(stop & ((1u << k9_ctz(free_match)) - 1u));
                if (below) lead_clip = 32u * w + 32u - k9_clz(below);
                break;
            }
            if (stop) lead_clip = 32u * w + 32u - k9_clz(stop);
        }
        trail_clip = read_size;
        for (uint32_t w = n_words; w-- > 0;)
        {
            uint32_t m, sc, cf;
            k9_word(v, a0, a1, best, range, maxScore, 32u * w, m, sc, cf);
            const uint32_t valid(read_size - 32u * w >= 32u ? 0xFFFFFFFFu : (1u << (read_size - 32u * w)) - 1u);
            const uint32_t free_match(m & ~cf & valid), stop((cf | sc) & valid);
            if (free_match)
            {
                const uint32_t above(stop & ~((2u << (31u - k9_clz(free_match))) - 1u));
                if (above) trail_clip = 32u * w + k9_ctz(above);
                break;
            }
            if (stop) trail_clip = 32u * w + k9_ctz(stop);
        }
        // leading_clip >= trailing_clip: clipping failed, finishRealignment reverts to the chosen alignment (:1432-1435)
        clip = (lead_clip < trail_clip) && (lead_clip != 0 || trail_clip != read_size);
    }
    k9_writer w = {slots, 0, cap, true};
    int32_t pos(b.aln_pos[best]);
    if (!clip)
    {
        for (uint32_t s = 0; s < n_path; ++s) k9_push(w, path[s].kind, path[s].len);
    }
    else // soft_clip_alignment, :255-338
    {
        uint32_t read_head(0);
        for (uint32_t s = 0; s < n_path; ++s)
        {
            const unsigned t(path[s].kind);
            const uint32_t len(path[s].len);
            if (k9_align_match(t) || t == SX_AP_INSERT)
            {
                if (lead_clip > read_head)
                {
                    const uint32_t c(len < lead_clip - read_head ? len : lead_clip - read_head);
                    k9_extend_or_add_sc(w, c);
                    if (k9_align_match(t)) pos += (int32_t)c;
                    if (c < len) k9_push(w, t, len - c);
                }
                else if (trail_clip < read_head + len)
                {
                    const uint32_t over(read_head + len - trail_clip);
                    const uint32_t c(len < over ? len : over);
                    if (c < len) k9_push(w, t, len - c);
                    k9_extend_or_add_sc(w, c);
                }
                else k9_push(w, t, len);
                read_head += len;
            }
            else if (t == SX_AP_DELETE || t == SX_AP_SKIP)
            {
                if (lead_clip >= read_head) pos += (int32_t)len;
                else if (trail_clip <= read_head)
                {
                }
                else k9_push(w, t, len);
            }
            else if (t == SX_AP_SOFT_CLIP)
            {
                k9_extend_or_add_sc(w, len);
                read_head += len;
            }
            else if (t == SX_AP_HARD_CLIP) k9_push(w, t, len);
            else return SX_REALIGN_ST_BADPATH;
        }
    }
    if (!w.ok) return SX_REALIGN_ST_BADPATH;
    for (uint32_t i = 0; i < w.n; ++i) slots[i].kind = k9_out_kind(b, slots[i].kind);
    for (uint32_t i = w.n; i < cap; ++i) slots[i] = sx_aln_seg{0, k9_out_kind(b, SX_AP_HARD_CLIP), 0};
    out_pos = pos;
    out_n = (uint16_t)w.n;
    return SX_REALIGN_ST_REALIGNED;
}

// a read without a realignment: its slots become no-op pads or, when the batch carries the mapper's alignments, that alignment
// (read_segment::getBestAlignment, starling_read_segment.hh:134-138)
K9_HD void k9_fallback(const sx_realign_batch& b, const uint32_t r, sx_aln_seg* slots, const uint32_t cap, int32_t& out_pos, uint16_t& out_n)
{
    uint32_t n(0);
    if (b.raw_seg_off)
    {
        const uint32_t s0(b.raw_seg_off[r]);
        n = b.raw_seg_off[r + 1] - s0;
        n = n < cap ? n : cap;
        for (uint32_t i = 0; i < n; ++i) slots[i] = sx_aln_seg{b.raw_segs[s0 + i].len, k9_out_kind(b, b.raw_segs[s0 + i].kind), 0};
        out_pos = b.raw_pos[r];
        out_n = (uint16_t)n;
    }
    for (uint32_t i = n; i < cap; ++i) slots[i] = sx_aln_seg{0, k9_out_kind(b, SX_AP_HARD_CLIP), 0};
}
