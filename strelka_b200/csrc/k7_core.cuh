// k7_core.cuh -- the per-read body of K7 enumerate_alignments (include/strelka_b200.h), written once for the device.
//
// The reference enumerates a read's candidate alignments with a recursion that passes ordered containers BY VALUE
// (starling_common/starling_read_align.cpp:857-878: indel_status_map, haplotypeStatusMap, indel_order, read_range, cal) and
// collects the results in a std::set<CandidateAlignment>.  Read closely, the containers are append-only along a search path:
//   * indel_order and indel_status_map always hold the same keys (every insertion into one is an insertion into the other:
//     add_indels_in_range :359-367, getCandidateAlignments :1895-1908); sort_remove_only_indels_last only permutes the entries
//     appended in the same call (:920, `current_depth` = the size before the call), so once a key has a position in indel_order it
//     keeps it for the whole subtree.  Hence ONE shared order[] array used as a stack (a child appends, the parent truncates) and
//     per-frame 64-bit masks indexed by that position for is_present / is_remove_only.
//   * the IndelBuffer window of the region is in IndelKey order, so "iterate the map" = ascending window index and IndelKey
//     comparisons are integer comparisons of window indices.
//   * the recursion becomes an explicit stack of frames with a resume stage (unchanged branch, start-pinned toggle, end-pinned
//     toggle); the std::set becomes a sorted index array over alignment slots with the set's own comparison.
//
// The functions are __host__ __device__ so that tests/cpp/k7_core_host.cpp can run exactly this code on the CPU against the
// reference's own getCandidateAlignments (a test of the device logic; the product has no host execution path -- k7_enumerate.cu
// only launches the kernels).
#pragma once

#include "strelka_b200.h"

#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define K7_HD __host__ __device__ __forceinline__
#define K7_HDN __host__ __device__ __noinline__
#else
#define K7_HD inline
#define K7_HDN inline
#endif

#define K7_MAX_INDELS 64u // indel_status_map entries of one read's search (64-bit masks)
#define K7_MAX_SEGS 32u   // path segments of one alignment
#define K7_MAX_KEYS 24u   // cal.getIndels() entries of one alignment
#define K7_MAX_HAP 4u     // active regions one read's search touches

struct k7_path // CandidateAlignment minus its indel set
{
    int32_t pos;
    uint16_t lead, trail; // window index or SX_NO_KEY
    uint32_t n_seg;
    uint32_t ref_len;     // apath_ref_length of seg[0..n_seg), kept up to date by k7_push_seg (the search asks for it at every call)
    uint32_t seg[K7_MAX_SEGS]; // one word per segment, sx_aln_seg's own bytes: len | kind << 16 | flags << 24 (kind = SX_AP_*); one load / store each
};

struct k7_cal // one element of the std::set<CandidateAlignment>; the key list sits in front of the (mostly empty) segment array so that an
{             // ordinary alignment -- two keys, five segments -- occupies one stretch of ~90 bytes instead of two 150 bytes apart
    uint32_t n_keys;
    uint16_t keys[K7_MAX_KEYS];
    k7_path p;
};

struct k7_hap // HaplotypeStatus of one active region (:134-179)
{
    int32_t id;
    int8_t c[SX_ENUM_MAX_SAMPLES];
    uint8_t any_on;
    uint8_t pad[3];
};

struct k7_frame // the by-value arguments of one candidate_alignment_search call + where to resume it
{
    uint64_t present, remove_only; // by position in order[]
    int32_t rr_begin, rr_end;      // read_range
    uint16_t n;                    // indel_order.size() == indel_status_map.size() in this call
    uint8_t depth, itd, ttd;       // depth, indelToggleDepth, totalToggleDepth
    uint8_t stage;                 // 0 entry, 1 after the unchanged branch, 2 after the start pin, 3 done
    int8_t mt;                     // max_read_indel_toggle
    uint8_t is_on;                 // isCurIndelOn at entry
    uint8_t cal_at;                // the frame whose `cal` is this call's alignment: a call that leaves the indel as it is shares its caller's
    uint32_t n_hap;
    k7_hap hap[K7_MAX_HAP];
    k7_path cal;
};

#define K7_ST_RETRY 0x80u // internal: the small (local-memory) scratch of the fast path is full; the read goes to the arena tier

struct k7_scratch // one thread's working memory (contiguous per thread)
{
    uint16_t* order;  // [K7_MAX_INDELS] window indices, the shared indel_order stack
    k7_frame* frames; // [maxF]
    k7_cal* slots;    // [maxA + 1]
    uint16_t* idx;    // [maxA] slots in std::set order
    uint32_t maxA;
    uint32_t maxF;    // frames available (K7_MAX_INDELS + 1 = as deep as a search can get)
    uint32_t full;    // status when a frame or an alignment slot is missing: SX_ENUM_ST_LIMIT, or K7_ST_RETRY for the small tier
    uint32_t n;       // alignments in the set
};

K7_HD constexpr size_t k7_scratch_bytes(const uint32_t maxA, const uint32_t maxF = K7_MAX_INDELS + 1)
{
    size_t b(0);
    b += ((size_t)K7_MAX_INDELS * 2 + 15) & ~(size_t)15;
    b += (sizeof(k7_frame) * maxF + 15) & ~(size_t)15;
    b += (sizeof(k7_cal) * ((size_t)maxA + 1) + 15) & ~(size_t)15;
    b += ((size_t)maxA * 2 + 15) & ~(size_t)15;
    return b;
}

K7_HD k7_scratch k7_scratch_at(unsigned char* base, const uint32_t maxA, const uint32_t maxF = K7_MAX_INDELS + 1, const uint32_t full = SX_ENUM_ST_LIMIT)
{
    k7_scratch S;
    size_t o(0);
    S.frames = reinterpret_cast<k7_frame*>(base + o);
    o += (sizeof(k7_frame) * maxF + 15) & ~(size_t)15;
    S.slots = reinterpret_cast<k7_cal*>(base + o);
    o += (sizeof(k7_cal) * ((size_t)maxA + 1) + 15) & ~(size_t)15;
    S.order = reinterpret_cast<uint16_t*>(base + o);
    o += ((size_t)K7_MAX_INDELS * 2 + 15) & ~(size_t)15;
    S.idx = reinterpret_cast<uint16_t*>(base + o);
    S.maxA = maxA;
    S.maxF = maxF;
    S.full = full;
    S.n = 0;
    return S;
}

struct k7_read // what the search reads of one read and its region
{
    const sx_indel_key* win;
    const sx_key_hap* hap; // or NULL
    uint32_t n_win;
    const uint16_t* use_keys;
    uint32_t n_use;
    int32_t realign_begin, realign_end;
    uint32_t read_length; // cal_read_length (:1933-1953)
    uint32_t hc_lead, hc_trail, sc_lead, sc_trail;
    const sx_enum_opts* opt;
};

K7_HD uint32_t k7_sw(const unsigned kind, const uint32_t len) { return len | ((uint32_t)kind << 16); }
K7_HD unsigned k7_sk(const uint32_t w) { return (w >> 16) & 0xFFu; }
K7_HD uint32_t k7_sl(const uint32_t w) { return w & 0xFFFFu; }
K7_HD uint32_t k7_seg_load(const sx_aln_seg* a) // (the arrays are 4-byte aligned: device allocations, numpy buffers)
{
    return (uint32_t)a->len | ((uint32_t)a->kind << 16) | ((uint32_t)a->flags << 24);
}
K7_HD bool k7_is_mismatch(const sx_indel_key& k) { return k.type == SX_INDEL_TYPE_MISMATCH; }
K7_HD int32_t k7_right(const sx_indel_key& k) { return k.pos + (int32_t)k.del_len; }
K7_HD bool k7_prim_del(const sx_indel_key& k) { return k.type == SX_INDEL_TYPE_INDEL && k.ins_len == 0 && k.del_len > 0; }

// indel_util.cpp:29-45
K7_HD bool k7_conflict(const sx_indel_key& a, const sx_indel_key& b)
{
    const int64_t margin((k7_is_mismatch(a) || k7_is_mismatch(b)) ? 0 : 1);
    const int64_t b1(a.pos), b2(b.pos);
    return (b2 + b.del_len + margin > b1) && (b2 < b1 + a.del_len + margin);
}

// indel_util.cpp:49-63; known_pos_range [b, e)
K7_HD bool k7_bp_intersect(const int32_t b, const int32_t e, const sx_indel_key& k)
{
    if (k7_is_mismatch(k)) return k.pos >= b && k.pos < e;
    if (k.pos > b && k.pos < e) return true;
    const int32_t r(k7_right(k));
    if (r == k.pos) return false;
    return r > b && r < e;
}

// indel_util.cpp:67-76
K7_HD bool k7_bp_adjacent(const int32_t b, const int32_t e, const sx_indel_key& k)
{
    if (k.pos + 1 > b && k.pos - 1 < e) return true;
    const int32_t r(k7_right(k));
    if (r == k.pos) return false;
    return r + 1 > b && r - 1 < e;
}

K7_HD bool k7_seg_read_len(const unsigned t) { return t == SX_AP_MATCH || t == SX_AP_INSERT || t == SX_AP_SOFT_CLIP || t == SX_AP_SEQ_MATCH || t == SX_AP_SEQ_MISMATCH; }
K7_HD bool k7_seg_ref_len(const unsigned t) { return t == SX_AP_MATCH || t == SX_AP_DELETE || t == SX_AP_SKIP || t == SX_AP_SEQ_MATCH || t == SX_AP_SEQ_MISMATCH; }
K7_HD bool k7_seg_unaligned_edge(const unsigned t) { return t == SX_AP_INSERT || t == SX_AP_HARD_CLIP || t == SX_AP_SOFT_CLIP; }

K7_HD uint32_t k7_ref_length_of(const k7_path& p) // apath_ref_length, align_path.cpp:160-169
{
    uint32_t v(0);
    for (uint32_t i = 0; i < p.n_seg; ++i)
        if (k7_seg_ref_len(k7_sk(p.seg[i]))) v += k7_sl(p.seg[i]);
    return v;
}
K7_HD uint32_t k7_ref_length(const k7_path& p) { return p.ref_len; }

K7_HD uint32_t k7_unaligned_prefix(const k7_path& p) // align_path.cpp:192-201
{
    uint32_t v(0);
    for (uint32_t i = 0; i < p.n_seg; ++i)
    {
        const uint32_t w(p.seg[i]);
        if (!k7_seg_unaligned_edge(k7_sk(w))) return v;
        if (k7_seg_read_len(k7_sk(w))) v += k7_sl(w);
    }
    return v;
}

K7_HD uint32_t k7_unaligned_suffix(const k7_path& p) // align_path.cpp:206-215
{
    uint32_t v(0);
    for (uint32_t i = p.n_seg; i-- > 0;)
    {
        const uint32_t w(p.seg[i]);
        if (!k7_seg_unaligned_edge(k7_sk(w))) return v;
        if (k7_seg_read_len(k7_sk(w))) v += k7_sl(w);
    }
    return v;
}

// get_soft_clip_alignment_range, alignment_util.cpp:45-55 (apath_insert_lead_size / trail_size, align_path.cpp:302-345)
K7_HD void k7_soft_clip_range(const k7_path& p, int32_t& b, int32_t& e)
{
    uint32_t lead(0), trail(0);
    for (uint32_t i = 0; i < p.n_seg; ++i)
    {
        const uint32_t w(p.seg[i]);
        const unsigned t(k7_sk(w));
        if (t == SX_AP_HARD_CLIP || t == SX_AP_SOFT_CLIP) continue;
        if (t != SX_AP_INSERT) break;
        lead += k7_sl(w);
    }
    for (uint32_t i = p.n_seg; i-- > 0;)
    {
        const uint32_t w(p.seg[i]);
        const unsigned t(k7_sk(w));
        if (t == SX_AP_HARD_CLIP || t == SX_AP_SOFT_CLIP) continue;
        if (t != SX_AP_INSERT) break;
        trail += k7_sl(w);
    }
    b = p.pos - (int32_t)lead;
    e = p.pos + (int32_t)k7_ref_length(p) + (int32_t)trail;
}

K7_HD bool k7_push_seg(k7_path& p, const unsigned kind, const uint32_t len)
{
    if (p.n_seg >= K7_MAX_SEGS || len > 0xFFFFu) return false;
    p.seg[p.n_seg] = k7_sw(kind, len);
    p.n_seg++;
    if (k7_seg_ref_len(kind)) p.ref_len += len;
    return true;
}

// the keys that are switched on, in IndelKey (= window index) order: `current_indels` (:1157-1161)
K7_HD uint32_t k7_present_sorted(const uint16_t* order, const uint32_t n, const uint64_t present, uint16_t* out)
{
    uint32_t m(0);
    for (uint32_t i = 0; i < n; ++i)
    {
        if (!((present >> i) & 1)) continue;
        const uint16_t k(order[i]);
        uint32_t j(m++);
        for (; j > 0 && out[j - 1] > k; --j) out[j] = out[j - 1];
        out[j] = k;
    }
    return m;
}

// make_start_pos_alignment, :393-584.  0 = ok, else SX_ENUM_ST_EXCEPTION (a throw, or an assert the reference would trip) or
// SX_ENUM_ST_LIMIT
#define K7_PUSH(kind, len)                                                      \
    do                                                                          \
    {                                                                           \
        const uint32_t k7_len_(len);                                            \
        if (ns >= K7_MAX_SEGS || k7_len_ > 0xFFFFu) return SX_ENUM_ST_LIMIT;    \
        cal.seg[ns++] = k7_sw(kind, k7_len_);                                   \
        if (k7_seg_ref_len(kind)) rl += k7_len_;                                \
    } while (0)
K7_HDN uint32_t k7_make_start_pos(const sx_indel_key* win, const int32_t ref_start, const int32_t read_start, const uint32_t read_length, const uint16_t* indels,
                                  const uint32_t n_indels, k7_path& cal)
{
    if (read_length == 0 || ref_start < 0 || read_start < 0) return SX_ENUM_ST_EXCEPTION;
    const bool is_leading_read(read_start != 0);
    cal.pos = ref_start;
    cal.lead = cal.trail = SX_NO_KEY;
    uint32_t ns(0), rl(0); // cal.n_seg / cal.ref_len, in registers until the path is complete
    int32_t ref_head(ref_start), read_head(read_start);
    bool prev_mismatch(false);
    for (uint32_t ii = 0; ii < n_indels; ++ii)
    {
        const uint16_t w(indels[ii]);
        const sx_indel_key ik(win[w]);
        const bool mismatch(k7_is_mismatch(ik));
        const int32_t right(k7_right(ik));
        if (right < ref_start) continue;
        if (right == ref_start)
        {
            if (mismatch) continue;
            if (!is_leading_read) continue;
        }
        const bool first(ns == 0);
        if (is_leading_read && first)
        {
            if (ik.pos != ref_start) return SX_ENUM_ST_EXCEPTION;                 // :440-458 "Anomalous condition for indel candidate"
            if (ik.ins_len == 0) return SX_ENUM_ST_EXCEPTION;                     // assert :461 (breakends are not sent)
            if ((int32_t)ik.ins_len < read_start) return SX_ENUM_ST_EXCEPTION;    // assert :466
            K7_PUSH(SX_AP_INSERT, (uint32_t)read_start);
            if (ik.del_len > 0)
            {
                K7_PUSH(SX_AP_DELETE, ik.del_len);
                ref_head += ik.del_len;
            }
            cal.lead = w;
            prev_mismatch = mismatch;
            continue;
        }
        if (first && read_start != 0) return SX_ENUM_ST_EXCEPTION; // assert :480
        const bool is_edge_delete(k7_prim_del(ik) && ik.pos == ref_start);
        const int32_t matchSegmentSize(ik.pos - ref_head);
        const int32_t minMatchSegmentSize((prev_mismatch || mismatch) ? 0 : 1);
        if (matchSegmentSize < minMatchSegmentSize && !is_edge_delete) return SX_ENUM_ST_EXCEPTION; // :487-493
        if (ik.pos < ref_head) return SX_ENUM_ST_EXCEPTION;                                         // assert :495
        const uint32_t match_segment((uint32_t)matchSegmentSize);
        if (!(first || match_segment > 0 || mismatch || prev_mismatch)) return SX_ENUM_ST_EXCEPTION; // assert :498
        if (((uint32_t)read_head + match_segment > read_length) || (((uint32_t)read_head + match_segment == read_length) && !k7_prim_del(ik))) break;
        if (match_segment > 0)
        {
            K7_PUSH(SX_AP_MATCH, match_segment);
            ref_head += (int32_t)match_segment;
            read_head += (int32_t)match_segment;
        }
        if (mismatch)
        {
            K7_PUSH(SX_AP_SEQ_MISMATCH, ik.del_len);
            ref_head += ik.del_len;
            read_head += ik.del_len;
            if (read_head >= (int32_t)read_length) break;
        }
        else if (ik.type == SX_INDEL_TYPE_INDEL)
        {
            if (ik.del_len > 0)
            {
                K7_PUSH(SX_AP_DELETE, ik.del_len);
                ref_head += ik.del_len;
            }
            if (ik.ins_len > 0)
            {
                const uint32_t max_insert_length(read_length - (uint32_t)read_head);
                const uint32_t insert_length(ik.ins_len < max_insert_length ? ik.ins_len : max_insert_length);
                K7_PUSH(SX_AP_INSERT, insert_length);
                read_head += (int32_t)insert_length;
                if (ik.ins_len >= max_insert_length)
                {
                    cal.trail = w;
                    break;
                }
            }
            else
            {
                if (match_segment == 0) cal.lead = w;
                else if (read_head == (int32_t)read_length) cal.trail = w;
            }
        }
        else return SX_ENUM_ST_EXCEPTION; // :568-572 "Unexpected indel state"
        prev_mismatch = mismatch;
    }
    if (read_head > (int32_t)read_length) return SX_ENUM_ST_EXCEPTION; // assert :577
    if (read_head < (int32_t)read_length)
    {
        K7_PUSH(SX_AP_MATCH, read_length - (uint32_t)read_head);
    }
    cal.n_seg = ns;
    cal.ref_len = rl;
    return 0;
}

#undef K7_PUSH

// get_end_pin_start_pos, :593-719
K7_HDN uint32_t k7_end_pin_start_pos(const sx_indel_key* win, const uint16_t* indels, const uint32_t n_indels, const uint32_t read_length, const int32_t ref_end,
                                     const int32_t read_end, int32_t& ref_start, int32_t& read_start)
{
    if (read_length == 0 || ref_end <= 0 || read_end <= 0) return SX_ENUM_ST_EXCEPTION; // asserts :602-604
    ref_start = ref_end;
    read_start = read_end;
    const bool is_trailing_read(read_end != (int32_t)read_length);
    bool is_first(true), prev_mismatch(false);
    for (uint32_t ii = n_indels; ii-- > 0;)
    {
        const sx_indel_key ik(win[indels[ii]]);
        const bool mismatch(k7_is_mismatch(ik));
        if (ik.pos > ref_end) continue;
        if (ik.pos == ref_end)
        {
            if (mismatch) continue;
            if (!is_trailing_read) continue;
        }
        const bool is_trailing_indel(!mismatch && k7_right(ik) == ref_end);
        if (is_trailing_indel)
        {
            if (!(is_first && ref_start == ref_end)) return SX_ENUM_ST_EXCEPTION; // assert :636
            if (ik.ins_len > 0 && ik.ins_len < read_length - (uint32_t)read_end) return SX_ENUM_ST_EXCEPTION; // assert :644
            ref_start -= (int32_t)ik.del_len;
        }
        else
        {
            if (is_first && read_end != (int32_t)read_length) return SX_ENUM_ST_EXCEPTION; // :652-658 "Unexpected realignment state"
            const int32_t matchSegmentSize(ref_start - k7_right(ik));
            const int32_t minMatchSegmentSize((prev_mismatch || mismatch) ? 0 : 1);
            if (matchSegmentSize < minMatchSegmentSize) return SX_ENUM_ST_EXCEPTION; // :670-676 "Unexpected indel position"
            const uint32_t match_segment((uint32_t)(matchSegmentSize < read_start ? matchSegmentSize : read_start));
            ref_start -= (int32_t)match_segment;
            read_start -= (int32_t)match_segment;
            if (read_start == 0) return 0;
            if (mismatch)
            {
                ref_start -= (int32_t)ik.del_len;
                read_start -= (int32_t)ik.del_len;
                if (read_start == 0) return 0;
            }
            else if (ik.type == SX_INDEL_TYPE_INDEL)
            {
                ref_start -= (int32_t)ik.del_len;
                if (ik.ins_len > 0)
                {
                    if ((int32_t)ik.ins_len >= read_start) return 0;
                    read_start -= (int32_t)ik.ins_len;
                }
            }
            else return SX_ENUM_ST_EXCEPTION; // :705-709
        }
        is_first = false;
        prev_mismatch = mismatch;
    }
    if (read_start < 0) return SX_ENUM_ST_EXCEPTION; // assert :716
    ref_start -= read_start;
    read_start = 0;
    return 0;
}

// CandidateAlignment::operator< (CandidateAlignment.hh:38-49) with alignment::operator< (alignment.hh:73-91; every alignment of a
// read has the read's strand) and path_segment::operator< (align_path.hh:190-196); std::set<IndelKey>::operator< is the
// lexicographic comparison of the window indices.  <0, 0, >0
K7_HD int k7_compare(const k7_cal& a, const k7_cal& b)
{
    if (a.p.pos != b.p.pos) return a.p.pos < b.p.pos ? -1 : 1;
    if (a.p.n_seg != b.p.n_seg) return a.p.n_seg < b.p.n_seg ? -1 : 1;
    for (uint32_t i = 0; i < a.p.n_seg; ++i)
    {
        const uint32_t wa(a.p.seg[i]), wb(b.p.seg[i]); // (flags are always 0 here)
        if (wa == wb) continue;
        if (k7_sk(wa) != k7_sk(wb)) return k7_sk(wa) < k7_sk(wb) ? -1 : 1;
        return k7_sl(wa) < k7_sl(wb) ? -1 : 1;
    }
    const uint32_t m(a.n_keys < b.n_keys ? a.n_keys : b.n_keys);
    for (uint32_t i = 0; i < m; ++i)
        if (a.keys[i] != b.keys[i]) return a.keys[i] < b.keys[i] ? -1 : 1;
    if (a.n_keys != b.n_keys) return a.n_keys < b.n_keys ? -1 : 1;
    // IndelKey() (type NONE at position 0) sorts before every real key
    const int la(a.p.lead == SX_NO_KEY ? -1 : (int)a.p.lead), lb(b.p.lead == SX_NO_KEY ? -1 : (int)b.p.lead);
    if (la != lb) return la < lb ? -1 : 1;
    const int ta(a.p.trail == SX_NO_KEY ? -1 : (int)a.p.trail), tb(b.p.trail == SX_NO_KEY ? -1 : (int)b.p.trail);
    if (ta != tb) return ta < tb ? -1 : 1;
    return 0;
}

K7_HD bool k7_add_key(k7_cal& c, const uint16_t w) // std::set<IndelKey>::insert
{
    uint32_t j(0);
    while (j < c.n_keys && c.keys[j] < w) ++j;
    if (j < c.n_keys && c.keys[j] == w) return true;
    if (c.n_keys >= K7_MAX_KEYS) return false;
    for (uint32_t i = c.n_keys; i > j; --i) c.keys[i] = c.keys[i - 1];
    c.keys[j] = w;
    c.n_keys++;
    return true;
}

// recursion terminus (:924-931) + the two post-passes of getCandidateAlignments (:1966-1993): keys, clips back on, range filter,
// cal_set.insert
K7_HDN uint32_t k7_emit(const k7_read& R, k7_scratch& S, const k7_frame& f, const k7_path& fcal)
{
    k7_cal& c(S.slots[S.n]); // slots has maxA + 1 entries: the candidate is built in place and kept only if it is new
    // addKeysToCandidateAlignment, :789-804
    const int32_t sb(fcal.pos), se(fcal.pos + (int32_t)k7_ref_length(fcal));
    c.n_keys = 0;
    for (uint32_t i = 0; i < f.n; ++i)
    {
        if (!((f.present >> i) & 1)) continue;
        const uint16_t w(S.order[i]);
        if (!k7_bp_intersect(sb, se, R.win[w])) continue;
        if (!k7_add_key(c, w)) return SX_ENUM_ST_LIMIT;
    }
    if (fcal.lead != SX_NO_KEY && !k7_add_key(c, fcal.lead)) return SX_ENUM_ST_LIMIT;
    if (fcal.trail != SX_NO_KEY && !k7_add_key(c, fcal.trail)) return SX_ENUM_ST_LIMIT;
    // apath_clip_adder, align_path.cpp:515-549
    // (the counters stay in registers: the path is written once, a word per segment; clips carry no reference length)
    {
        const uint32_t n_in(fcal.n_seg);
        const uint32_t extra((R.hc_lead ? 1u : 0u) + (R.sc_lead ? 1u : 0u) + (R.sc_trail ? 1u : 0u) + (R.hc_trail ? 1u : 0u));
        if (n_in + extra > K7_MAX_SEGS || R.hc_lead > 0xFFFFu || R.sc_lead > 0xFFFFu || R.sc_trail > 0xFFFFu || R.hc_trail > 0xFFFFu) return SX_ENUM_ST_LIMIT;
        uint32_t m(0);
        if (R.hc_lead) c.p.seg[m++] = k7_sw(SX_AP_HARD_CLIP, R.hc_lead);
        if (R.sc_lead) c.p.seg[m++] = k7_sw(SX_AP_SOFT_CLIP, R.sc_lead);
        for (uint32_t i = 0; i < n_in; ++i) c.p.seg[m++] = fcal.seg[i];
        if (R.sc_trail) c.p.seg[m++] = k7_sw(SX_AP_SOFT_CLIP, R.sc_trail);
        if (R.hc_trail) c.p.seg[m++] = k7_sw(SX_AP_HARD_CLIP, R.hc_trail);
        c.p.pos = fcal.pos;
        c.p.lead = fcal.lead;
        c.p.trail = fcal.trail;
        c.p.n_seg = m;
        c.p.ref_len = fcal.ref_len;
    }
    // is_alignment_spanned_by_range, :1455-1459
    if (!(sb >= R.realign_begin && se <= R.realign_end)) return 0;
    // std::set::insert
    uint32_t lo(0), hi(S.n);
    while (lo < hi)
    {
        const uint32_t mid((lo + hi) / 2);
        const int cmp(k7_compare(S.slots[S.idx[mid]], c));
        if (cmp == 0) return 0;
        if (cmp < 0) lo = mid + 1;
        else hi = mid;
    }
    if (S.n >= S.maxA) return S.full;
    for (uint32_t i = S.n; i > lo; --i) S.idx[i] = S.idx[i - 1];
    S.idx[lo] = (uint16_t)S.n;
    S.n++;
    return 0;
}

K7_HD bool k7_usable(const k7_read& R, const uint16_t w) // is_usable_indel, :289-305
{
    if (R.win[w].flags & SX_IKF_CANDIDATE) return true;
    for (uint32_t i = 0; i < R.n_use; ++i)
        if (R.use_keys[i] == w) return true;
    return false;
}

// add_indels_in_range, :311-375, appending to order[0..n); new entries are never present.  0 or a status bit
K7_HDN uint32_t k7_add_indels_in_range(const k7_read& R, uint16_t* order, uint32_t& n, uint64_t& remove_only, const int32_t b, const int32_t e)
{
    // IndelBuffer::rangeIterator(b, e), IndelBuffer.cpp:76-91
    uint32_t k(0);
    {
        uint32_t lo(0), hi(R.n_win); // lower_bound(IndelKey(b - maxIndelSize)): first entry with pos >= b - maxIndelSize
        const int64_t want((int64_t)b - (int64_t)R.opt->max_indel_size);
        while (lo < hi)
        {
            const uint32_t mid((lo + hi) / 2);
            if ((int64_t)R.win[mid].pos < want) lo = mid + 1;
            else hi = mid;
        }
        k = lo;
    }
    for (; k < R.n_win && R.win[k].pos < e; ++k)
        if (k7_right(R.win[k]) >= b) break;
    for (; k < R.n_win && R.win[k].pos < e; ++k)
    {
        const sx_indel_key ik(R.win[k]);
        if (ik.type > SX_INDEL_TYPE_MISMATCH) return SX_ENUM_ST_LIMIT; // breakends are not sent
        if (!k7_bp_adjacent(b, e, ik)) continue;
        const bool is_remove_only(!k7_bp_intersect(b, e, ik));
        uint32_t at(n);
        for (uint32_t i = 0; i < n; ++i)
            if (order[i] == k)
            {
                at = i;
                break;
            }
        if (at < n)
        {
            if (!is_remove_only) remove_only &= ~((uint64_t)1 << at);
        }
        else if (k7_usable(R, (uint16_t)k))
        {
            if (n >= K7_MAX_INDELS) return SX_ENUM_ST_LIMIT;
            order[n] = (uint16_t)k;
            if (is_remove_only) remove_only |= ((uint64_t)1 << n);
            else remove_only &= ~((uint64_t)1 << n);
            n++;
        }
    }
    return 0;
}

// sort_remove_only_indels_last, :724-749, on order[start..n): entries that are present or not remove-only first (stable).  The
// mask bits travel with their entries.
K7_HD void k7_sort_remove_only_last(uint16_t* order, const uint32_t start, const uint32_t n, uint64_t& present, uint64_t& remove_only, uint64_t* inorig)
{
    if (n - start < 2) return;
    uint16_t tmp[K7_MAX_INDELS];
    uint64_t p2(0), r2(0), o2(0);
    uint32_t m(0);
    for (int pass = 0; pass < 2; ++pass)
        for (uint32_t i = start; i < n; ++i)
        {
            const bool pr((present >> i) & 1), ro((remove_only >> i) & 1);
            const bool firstGroup(pr || !ro);
            if (firstGroup != (pass == 0)) continue;
            tmp[m] = order[i];
            if (pr) p2 |= (uint64_t)1 << (start + m);
            if (ro) r2 |= (uint64_t)1 << (start + m);
            if (inorig && ((*inorig >> i) & 1)) o2 |= (uint64_t)1 << (start + m);
            m++;
        }
    const uint64_t keep(start == 0 ? 0 : (((uint64_t)1 << start) - 1));
    for (uint32_t i = 0; i < m; ++i) order[start + i] = tmp[i];
    present = (present & keep) | p2;
    remove_only = (remove_only & keep) | r2;
    if (inorig) *inorig = (*inorig & keep) | o2;
}

// getUpdatedSampleHaplotypeConstraints, :66-130
K7_HD int k7_updated_constraints(const int hc, const int curId, const bool isOn, const bool anyOn)
{
    if (hc < 0) return hc;
    if (curId < 0 && isOn) return -1;
    if (curId <= 0) return hc;
    const int fromCur(isOn ? curId : (3 - curId));
    switch (fromCur)
    {
    case 0: return anyOn ? -1 : 0;
    case 1:
    case 2:
        if (hc == 3 || hc == fromCur) return fromCur;
        return anyOn ? -1 : 0;
    default: // 3
        return hc > 0 ? hc : -1;
    }
}

// HaplotypeStatus::updateHaplotypeStatus, :146-170
K7_HD bool k7_update_hap(k7_hap& h, const int* ids, const bool isOn, const uint32_t n_samples)
{
    h.any_on = (h.any_on || isOn) ? 1 : 0;
    bool valid(false);
    for (uint32_t s = 0; s < n_samples; ++s)
    {
        const int u(k7_updated_constraints(h.c[s], ids[s], isOn, h.any_on != 0));
        if (u >= 0) valid = true;
        h.c[s] = (int8_t)u;
    }
    return valid;
}

K7_HD void k7_copy_path(k7_path& d, const k7_path& s)
{
    d.pos = s.pos;
    d.lead = s.lead;
    d.trail = s.trail;
    d.n_seg = s.n_seg;
    d.ref_len = s.ref_len;
    for (uint32_t i = 0; i < s.n_seg; ++i) d.seg[i] = s.seg[i];
}

// a child call: every by-value argument copied from the caller's frame as it stands now
K7_HD void k7_push_child(k7_frame& c, const k7_frame& f, const uint32_t itd, const uint32_t ttd)
{
    c.present = f.present;
    c.remove_only = f.remove_only;
    c.rr_begin = f.rr_begin;
    c.rr_end = f.rr_end;
    c.n = f.n;
    c.depth = (uint8_t)(f.depth + 1);
    c.itd = (uint8_t)itd;
    c.ttd = (uint8_t)ttd;
    c.stage = 0;
    c.mt = f.mt;
    c.is_on = 0;
    c.n_hap = f.n_hap;
    for (uint32_t i = 0; i < f.n_hap; ++i) c.hap[i] = f.hap[i];
}

// candidate_alignment_search, :857-1277, from the root frame S.frames[0] (already filled).  Returns the status bits of the read.
K7_HDN uint32_t k7_search(const k7_read& R, k7_scratch& S, const uint64_t inorig)
{
    uint32_t status(0);
    const sx_enum_opts& opt(*R.opt);
    int sp(0);
    while (sp >= 0)
    {
        k7_frame& f(S.frames[sp]);
        const k7_path& cal(S.frames[f.cal_at].cal);
        if (f.stage == 0)
        {
            // ---- new indel overlaps, :888-922
            bool is_new_indels(f.itd == 0);
            uint32_t n(f.n);
            {
                const uint32_t start_size(n);
                int32_t pb, pe;
                k7_soft_clip_range(cal, pb, pe);
                if (!(pb >= R.realign_begin && pe <= R.realign_end))
                {
                    --sp;
                    continue;
                }
                if (pb < f.rr_begin)
                {
                    const uint32_t st(k7_add_indels_in_range(R, S.order, n, f.remove_only, pb, f.rr_begin + 1));
                    if (st) return status | st;
                    f.rr_begin = pb;
                }
                if (pe > f.rr_end)
                {
                    const uint32_t st(k7_add_indels_in_range(R, S.order, n, f.remove_only, f.rr_end - 1, pe));
                    if (st) return status | st;
                    f.rr_end = pe;
                }
                if (!is_new_indels) is_new_indels = (start_size != n);
                // new entries are not present: clear any stale bit a sibling subtree left at these positions
                for (uint32_t i = start_size; i < n; ++i) f.present &= ~((uint64_t)1 << i);
                if (is_new_indels) k7_sort_remove_only_last(S.order, start_size, n, f.present, f.remove_only, nullptr);
                f.n = (uint16_t)n;
            }
            // ---- recursion terminus, :924-931
            if (f.depth == n)
            {
                const uint32_t st(k7_emit(R, S, f, cal));
                if (st) return status | st;
                --sp;
                continue;
            }
            // ---- toggle limits, :933-974
            if (is_new_indels)
            {
                const double max_indels(R.read_length * opt.max_candidate_indel_density);
                int mt((double)n > max_indels ? 1 : opt.max_read_indel_toggle);
                const int max_toggle(n >= opt.n_max_toggle ? 1 : (int)opt.max_toggle[n]);
                if (max_toggle < mt) mt = max_toggle;
                f.mt = (int8_t)mt;
            }
            if ((int)f.itd > (int)f.mt)
            {
                status |= SX_ENUM_ST_MAX_TOGGLE;
                --sp;
                continue;
            }
        }
        // ---- the current indel and what is already switched on before it, :994-1041 (recomputed at every resume: cheap and
        // it keeps the frame small)
        const uint32_t n(f.n);
        const uint16_t curW(S.order[f.depth]);
        const sx_indel_key cur(R.win[curW]);
        const bool curMismatch(k7_is_mismatch(cur));
        bool conflicting(false), containsNotDiscovered(false);
        {
            // at stage >= 1 the current indel's own bit may be toggled; positions < depth are untouched
            for (uint32_t i = 0; i < f.depth; ++i)
            {
                if (!((f.present >> i) & 1)) continue;
                const sx_indel_key ik(R.win[S.order[i]]);
                if (k7_conflict(ik, cur)) conflicting = true;
                if (ik.flags & SX_IKF_NOT_DISCOVERED) containsNotDiscovered = true;
            }
        }
        const uint32_t n_samples(opt.n_samples);
        const sx_key_hap* kh(R.hap ? R.hap + curW : nullptr);
        const int32_t curAr(kh ? kh->active_region_id : -1);
        const bool inAr(curAr >= 0);
        const bool curNotDiscovered((cur.flags & SX_IKF_NOT_DISCOVERED) != 0);
        int ids[SX_ENUM_MAX_SAMPLES] = {0, 0, 0, 0};
        uint32_t arSlot(0);
        if (f.stage == 0)
        {
            f.is_on = (uint8_t)((f.present >> f.depth) & 1);
            if (inAr)
            {
                uint32_t i(0);
                for (; i < f.n_hap; ++i)
                    if (f.hap[i].id == curAr) break;
                if (i == f.n_hap)
                {
                    if (f.n_hap >= K7_MAX_HAP) return status | SX_ENUM_ST_LIMIT;
                    f.hap[i].id = curAr;
                    for (uint32_t s = 0; s < SX_ENUM_MAX_SAMPLES; ++s) f.hap[i].c[s] = 3;
                    f.hap[i].any_on = 0;
                    f.n_hap++;
                }
            }
        }
        const bool isOn(f.is_on != 0);
        if (inAr)
        {
            for (arSlot = 0; arSlot < f.n_hap; ++arSlot)
                if (f.hap[arSlot].id == curAr) break;
            // getCurIndelHaplotypeIds, :811-849
            const bool inOriginal((inorig >> f.depth) & 1);
            for (uint32_t s = 0; s < n_samples; ++s)
            {
                int id(kh->haplotype_id[s]);
                if (id == 0)
                {
                    bool validHere(!opt.is_haplotyping_enabled || ((kh->bypass_mask >> s) & 1) || (cur.flags & SX_IKF_FORCED_OUTPUT));
                    if (!validHere && s == opt.sample_id && inOriginal) validHere = true;
                    if (curMismatch && s != opt.sample_id) validHere = false;
                    id = validHere ? 0 : -1;
                }
                ids[s] = id;
            }
        }

        if ((uint32_t)sp + 1 >= S.maxF) return status | S.full; // no frame left for a child call (only the small tier can get here)
        if (f.stage == 0)
        {
            // ---- alignment 1: unchanged, :1043-1096
            f.stage = 1;
            k7_frame& c(S.frames[sp + 1]);
            k7_push_child(c, f, f.itd, f.ttd);
            bool valid(true);
            if (!conflicting && inAr) valid = k7_update_hap(c.hap[arSlot], ids, isOn, n_samples);
            else valid = !curMismatch || !isOn;
            if (isOn && containsNotDiscovered && curNotDiscovered) valid = false;
            if (!valid && f.ttd == 0) valid = true;
            if (valid)
            {
                c.cal_at = f.cal_at; // the same alignment: nothing to copy
                ++sp;
                continue;
            }
        }
        if (f.stage == 1)
        {
            // ---- may the indel be toggled at all?  :1098-1147
            f.stage = 2;
            k7_frame& c(S.frames[sp + 1]);
            k7_push_child(c, f, 0, 0);
            bool valid(true);
            if (!conflicting && inAr) valid = k7_update_hap(c.hap[arSlot], ids, !isOn, n_samples);
            else valid = !curMismatch || isOn;
            if (!isOn && containsNotDiscovered && curNotDiscovered) valid = false;
            bool go(valid);
            if (go && !isOn)
            {
                if ((f.remove_only >> f.depth) & 1) go = false;
                if (conflicting) go = false;
            }
            const uint32_t inc(curMismatch ? 0 : 1);
            if (go && (int)(f.itd + inc) > (int)f.mt)
            {
                status |= SX_ENUM_ST_MAX_TOGGLE;
                go = false;
            }
            if (!go)
            {
                --sp;
                continue;
            }
            // ---- changed cases, :1149-1161
            if (isOn) f.present &= ~((uint64_t)1 << f.depth);
            else f.present |= ((uint64_t)1 << f.depth);
            // ---- alignment 2: start pin, :1170-1219
            const int32_t ref_start(cal.pos);
            bool start_pin_valid(true);
            if (!curMismatch)
            {
                const bool delete_span(cur.pos <= ref_start && ref_start < k7_right(cur));
                const bool indel_span(isOn && curW == cal.lead);
                start_pin_valid = !(delete_span || indel_span);
            }
            if (start_pin_valid)
            {
                uint16_t cur_indels[K7_MAX_INDELS];
                const uint32_t n_cur(k7_present_sorted(S.order, n, f.present, cur_indels));
                const int32_t read_start((int32_t)k7_unaligned_prefix(cal));
                const uint32_t st(k7_make_start_pos(R.win, ref_start, read_start, R.read_length, cur_indels, n_cur, c.cal));
                if (st) return status | st;
                k7_push_child(c, f, f.itd + inc, f.ttd + 1u);
                c.cal_at = (uint8_t)(sp + 1);
                if (!conflicting && inAr) k7_update_hap(c.hap[arSlot], ids, !isOn, n_samples);
                ++sp;
                continue;
            }
        }
        if (f.stage == 2)
        {
            f.stage = 3;
            // ---- alignment 3: end pin, :1221-1276
            if (curMismatch || cur.del_len == cur.ins_len)
            {
                --sp;
                continue;
            }
            const int32_t ref_end(cal.pos + (int32_t)k7_ref_length(cal));
            const bool delete_span(cur.pos <= ref_end - 1 && ref_end - 1 < k7_right(cur));
            const bool indel_span(isOn && curW == cal.trail);
            if (!(delete_span || indel_span))
            {
                uint16_t cur_indels[K7_MAX_INDELS];
                const uint32_t n_cur(k7_present_sorted(S.order, n, f.present, cur_indels));
                const int32_t read_end((int32_t)R.read_length - (int32_t)k7_unaligned_suffix(cal));
                int32_t ref_start(0), read_start(0);
                uint32_t st(k7_end_pin_start_pos(R.win, cur_indels, n_cur, R.read_length, ref_end, read_end, ref_start, read_start));
                if (st) return status | st;
                if (ref_start < 0) status |= SX_ENUM_ST_ORIGIN_SKIP;
                else
                {
                    k7_frame& c(S.frames[sp + 1]);
                    st = k7_make_start_pos(R.win, ref_start, read_start, R.read_length, cur_indels, n_cur, c.cal);
                    if (st) return status | st;
                    const uint32_t inc(1);
                    k7_push_child(c, f, f.itd + inc, f.ttd + 1u);
                    c.cal_at = (uint8_t)(sp + 1);
                    if (!conflicting && inAr) k7_update_hap(c.hap[arSlot], ids, !isOn, n_samples);
                    ++sp;
                    continue;
                }
            }
        }
        --sp;
    }
    return status;
}

struct k7_view
{
    sx_enum_batch b;
};

K7_HDN uint32_t k7_enumerate_read_raw(const k7_view& v, const uint32_t region, const uint32_t r, k7_scratch& S);

// getCandidateAlignments, :1816-1994, for read r of `region`: fills S (the set), returns the read's status bits.  A read that failed
// (SX_ENUM_ST_EXCEPTION / SX_ENUM_ST_LIMIT) reports that bit alone: the warnings collected before the failure are meaningless.
K7_HD uint32_t k7_enumerate_read(const k7_view& v, const uint32_t region, const uint32_t r, k7_scratch& S)
{
    const uint32_t st(k7_enumerate_read_raw(v, region, r, S));
    if (st & K7_ST_RETRY) return K7_ST_RETRY;
    const uint32_t fail(st & (SX_ENUM_ST_EXCEPTION | SX_ENUM_ST_LIMIT));
    return fail ? fail : st;
}

K7_HDN uint32_t k7_enumerate_read_raw(const k7_view& v, const uint32_t region, const uint32_t r, k7_scratch& S)
{
    const sx_enum_batch& b(v.b);
    S.n = 0;
    if (b.gate && !(b.gate[r] & SX_GATE_REALIGN)) return 0; // realignAndScoreRead returned before the search (K7g)
    k7_read R;
    const uint32_t k0(b.region_key_off[region]);
    R.win = b.keys + k0;
    R.hap = b.key_hap ? b.key_hap + k0 : nullptr;
    R.n_win = b.region_key_off[region + 1] - k0;
    R.use_keys = b.use_keys + b.use_key_off[r];
    R.n_use = b.use_key_off[r + 1] - b.use_key_off[r];
    R.realign_begin = b.realign_begin[region];
    R.realign_end = b.realign_end[region];
    R.opt = &b.opts;
    R.hc_lead = R.hc_trail = R.sc_lead = R.sc_trail = 0;
    const uint32_t read_length(b.read_len[r]);
    if (b.opts.n_samples == 0 || b.opts.n_samples > SX_ENUM_MAX_SAMPLES || b.opts.sample_id >= b.opts.n_samples) return SX_ENUM_ST_LIMIT;

    k7_frame& f(S.frames[0]);
    // getCandidateAlignment, :1481-1522 (the edge keys come from the host, which holds the read bases)
    {
        const uint32_t s0(b.in_seg_off[r]), ns(b.in_seg_off[r + 1] - s0);
        if (ns > K7_MAX_SEGS) return SX_ENUM_ST_LIMIT;
        f.cal.pos = b.in_pos[r];
        f.cal.lead = b.in_lead_key[r];
        f.cal.trail = b.in_trail_key[r];
        f.cal.n_seg = ns;
        for (uint32_t i = 0; i < ns; ++i) f.cal.seg[i] = k7_seg_load(b.in_segs + s0 + i);
        f.cal.ref_len = k7_ref_length_of(f.cal);
    }
    // indel set of the exemplar, :1843-1845
    int32_t eb, ee;
    k7_soft_clip_range(f.cal, eb, ee);
    uint32_t n(0);
    uint64_t present(0), remove_only(0), inorig(0);
    {
        const uint32_t st(k7_add_indels_in_range(R, S.order, n, remove_only, eb, ee));
        if (st) return st;
    }
    // mark what the input alignment already contains, :1853-1893
    bool recompute(false);
    uint16_t valid[K7_MAX_INDELS];
    uint32_t n_valid(0);
    for (uint32_t i = b.in_key_off[r]; i < b.in_key_off[r + 1]; ++i)
    {
        const uint16_t w(b.in_keys[i]);
        if (w == SX_NO_KEY) return SX_ENUM_ST_EXCEPTION; // an indel of the alignment that the window does not hold: what :1866-1872 throws for
        if (w >= R.n_win) return SX_ENUM_ST_LIMIT;
        uint32_t at(n);
        for (uint32_t j = 0; j < n; ++j)
            if (S.order[j] == w)
            {
                at = j;
                break;
            }
        const bool mismatch(k7_is_mismatch(R.win[w]));
        if (at == n)
        {
            if (mismatch) continue;
            return SX_ENUM_ST_EXCEPTION; // :1866-1872 "Exemplar alignment contains indel not found in the overlap indel set"
        }
        if (mismatch) recompute = true;
        present |= (uint64_t)1 << at;
        inorig |= (uint64_t)1 << at;
        if (n_valid < K7_MAX_INDELS) valid[n_valid++] = w; // in_keys ascend, so this is the set's order
    }
    if (recompute)
    {
        k7_path tmp;
        const uint32_t st(k7_make_start_pos(R.win, f.cal.pos, (int32_t)k7_unaligned_prefix(f.cal), read_length, valid, n_valid, tmp));
        if (st) return st;
        k7_copy_path(f.cal, tmp);
    }
    // indel_order: present entries first, each group in key order (:1895-1908) -- add_indels_in_range appended in key order --
    // then the non-present remove-only entries last (:1911)
    {
        uint16_t tmp[K7_MAX_INDELS];
        uint64_t p2(0), r2(0), o2(0);
        uint32_t m(0);
        for (int pass = 0; pass < 2; ++pass)
            for (uint32_t i = 0; i < n; ++i)
            {
                const bool pr((present >> i) & 1);
                if (pr != (pass == 0)) continue;
                tmp[m] = S.order[i];
                if (pr) p2 |= (uint64_t)1 << m;
                if ((remove_only >> i) & 1) r2 |= (uint64_t)1 << m;
                if ((inorig >> i) & 1) o2 |= (uint64_t)1 << m;
                m++;
            }
        for (uint32_t i = 0; i < n; ++i) S.order[i] = tmp[i];
        present = p2;
        remove_only = r2;
        inorig = o2;
        k7_sort_remove_only_last(S.order, 0, n, present, remove_only, &inorig);
    }
    // clips come off for the search and go back on afterwards, :1933-1953 (apath_clip_clipper, align_path.cpp:464-510)
    uint32_t cal_read_length(read_length);
    {
        const uint32_t ns(f.cal.n_seg);
        const bool clipped(ns > 0 && (k7_sk(f.cal.seg[0]) == SX_AP_SOFT_CLIP || k7_sk(f.cal.seg[0]) == SX_AP_HARD_CLIP ||
                                      (ns > 1 && (k7_sk(f.cal.seg[ns - 1]) == SX_AP_SOFT_CLIP || k7_sk(f.cal.seg[ns - 1]) == SX_AP_HARD_CLIP))));
        if (clipped)
        {
            bool is_lead(true);
            uint32_t m(0);
            for (uint32_t i = 0; i < ns; ++i)
            {
                const uint32_t sg(f.cal.seg[i]);
                if (k7_sk(sg) == SX_AP_HARD_CLIP) (is_lead ? R.hc_lead : R.hc_trail) += k7_sl(sg);
                else if (k7_sk(sg) == SX_AP_SOFT_CLIP) (is_lead ? R.sc_lead : R.sc_trail) += k7_sl(sg);
                else
                {
                    is_lead = false;
                    if (R.hc_trail || R.sc_trail) return SX_ENUM_ST_EXCEPTION; // asserts align_path.cpp:504-505
                    f.cal.seg[m++] = sg;
                }
            }
            f.cal.n_seg = m; // (clips carry no reference length: ref_len stands)
            if (cal_read_length < R.sc_lead + R.sc_trail) return SX_ENUM_ST_EXCEPTION; // assert :1950
            cal_read_length -= R.sc_lead + R.sc_trail;
        }
    }
    R.read_length = cal_read_length;
    f.present = present;
    f.remove_only = remove_only;
    f.rr_begin = eb;
    f.rr_end = ee;
    f.n = (uint16_t)n;
    f.depth = 0;
    f.itd = 0;
    f.ttd = 0;
    f.stage = 0;
    f.mt = (int8_t)b.opts.max_read_indel_toggle;
    f.is_on = 0;
    f.cal_at = 0;
    f.n_hap = 0;
    return k7_search(R, S, inorig);
}

// what a read contributes to the CSR output: alignments, segments, keys (0 for a failed read)
K7_HD void k7_count(const k7_scratch& S, const uint32_t status, uint32_t& n_aln, uint32_t& n_seg, uint32_t& n_key)
{
    n_aln = n_seg = n_key = 0;
    if (status & (SX_ENUM_ST_EXCEPTION | SX_ENUM_ST_LIMIT | K7_ST_RETRY)) return;
    n_aln = S.n;
    for (uint32_t i = 0; i < S.n; ++i)
    {
        n_seg += S.slots[i].p.n_seg;
        n_key += S.slots[i].n_keys;
    }
}

// write the set, in its order, at the read's offsets (aln_seg_off / aln_key_off get the START of each alignment; the batch-wide
// last entry is written by the caller)
K7_HD void k7_write(const k7_scratch& S, const sx_enum_out& o, const uint32_t a0, uint32_t s0, uint32_t k0)
{
    for (uint32_t i = 0; i < S.n; ++i)
    {
        const k7_cal& c(S.slots[S.idx[i]]);
        const uint32_t a(a0 + i);
        o.aln_pos[a] = c.p.pos;
        o.aln_lead_key[a] = c.p.lead;
        o.aln_trail_key[a] = c.p.trail;
        o.aln_seg_off[a] = s0;
        o.aln_key_off[a] = k0;
        for (uint32_t j = 0; j < c.p.n_seg; ++j) o.segs[s0 + j] = sx_aln_seg{(uint16_t)k7_sl(c.p.seg[j]), (uint8_t)k7_sk(c.p.seg[j]), (uint8_t)(c.p.seg[j] >> 24)};
        for (uint32_t j = 0; j < c.n_keys; ++j) o.aln_keys[k0 + j] = c.keys[j];
        s0 += c.p.n_seg;
        k0 += c.n_keys;
    }
}

// ---- the fast path's result log: a read's set as one blob of 32-bit words, in set order:
//   per alignment  [pos] [lead | trail << 16] [n_seg | n_keys << 8] [segs: n_seg words] [keys: ceil(n_keys / 2) words]
K7_HD uint32_t k7_blob_words(const k7_scratch& S)
{
    uint32_t w(0);
    for (uint32_t i = 0; i < S.n; ++i) w += 3u + S.slots[i].p.n_seg + (S.slots[i].n_keys + 1u) / 2u;
    return w;
}

K7_HD void k7_blob_write(const k7_scratch& S, uint32_t* dst)
{
    for (uint32_t i = 0; i < S.n; ++i)
    {
        const k7_cal& c(S.slots[S.idx[i]]);
        *dst++ = (uint32_t)c.p.pos;
        *dst++ = (uint32_t)c.p.lead | ((uint32_t)c.p.trail << 16);
        *dst++ = c.p.n_seg | (c.n_keys << 8);
        for (uint32_t j = 0; j < c.p.n_seg; ++j) *dst++ = c.p.seg[j];
        for (uint32_t j = 0; j < c.n_keys; j += 2) *dst++ = (uint32_t)c.keys[j] | ((j + 1 < c.n_keys ? (uint32_t)c.keys[j + 1] : 0u) << 16);
    }
}

// blob -> the read's place in the CSR output (what k7_write does from the scratch)
K7_HD void k7_blob_gather(const uint32_t* src, const uint32_t n_aln, const sx_enum_out& o, const uint32_t a0, uint32_t s0, uint32_t k0)
{
    for (uint32_t i = 0; i < n_aln; ++i)
    {
        const uint32_t a(a0 + i);
        o.aln_pos[a] = (int32_t)src[0];
        o.aln_lead_key[a] = (uint16_t)(src[1] & 0xFFFFu);
        o.aln_trail_key[a] = (uint16_t)(src[1] >> 16);
        const uint32_t ns(src[2] & 0xFFu), nk(src[2] >> 8);
        src += 3;
        o.aln_seg_off[a] = s0;
        o.aln_key_off[a] = k0;
        for (uint32_t j = 0; j < ns; ++j)
        {
            const uint32_t w(*src++);
            o.segs[s0 + j] = sx_aln_seg{(uint16_t)(w & 0xFFFFu), (uint8_t)((w >> 16) & 0xFFu), (uint8_t)(w >> 24)};
        }
        for (uint32_t j = 0; j < nk; j += 2)
        {
            const uint32_t w(*src++);
            o.aln_keys[k0 + j] = (uint16_t)(w & 0xFFFFu);
            if (j + 1 < nk) o.aln_keys[k0 + j + 1] = (uint16_t)(w >> 16);
        }
        s0 += ns;
        k0 += nk;
    }
}
