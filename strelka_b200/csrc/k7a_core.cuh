// k7a_core.cuh -- the per-read body of K7a alignment_indels (include/strelka_b200.h): which window entries a read's input alignment
// already contains.  Restates getAlignmentIndels(cal, ref, rseg, maxIndelSize, includeMismatches = true)
// (starling_common/CandidateAlignment.cpp:58-173) and the edge keys of getCandidateAlignment (starling_read_align.cpp:1481-1522) on
// K1's read / reference pools, with IndelKeys as window indices.  __host__ __device__: tests/cpp/k7a_core_host.cpp runs exactly this
// code on the CPU against the reference's own functions.
#pragma once

#include "strelka_b200.h"

#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define K7A_HD __host__ __device__ __forceinline__
#else
#define K7A_HD inline
#endif

#define K7A_MAX_KEYS 64u // keys of one input alignment (indels + window mismatches); more: the surplus is reported as SX_NO_KEY

struct k7a_view
{
    sx_enum_batch b;
    const sx_region* regions;
    const uint8_t* seq4;
    const char* ref;
    const uint32_t* key_ins_off;
    const char* key_ins;
};

K7A_HD uint8_t k7a_code(const uint8_t* seq4, const uint64_t read_byte, const uint32_t i) // bam_seq::get_code
{
    const uint8_t v(seq4[read_byte + (i >> 1)]);
    return (i & 1) ? (uint8_t)(v & 15) : (uint8_t)(v >> 4);
}
K7A_HD char k7a_char(const uint8_t c) // get_bam_seq_char, htsapi/bam_seq.hh:50-71
{
    return c == 0 ? '=' : c == 1 ? 'A' : c == 2 ? 'C' : c == 4 ? 'G' : c == 8 ? 'T' : 'N';
}
K7A_HD uint8_t k7a_ref_code(const k7a_view& v, const sx_region& g, const int32_t pos) // rc_segment_bam_seq::get_code: get_bam_seq_code(ref.get_base(pos))
{
    const int64_t i((int64_t)pos - g.ref_begin);
    const char c((i >= 0 && i < (int64_t)g.ref_len) ? v.ref[g.ref_off + (uint64_t)i] : 'N');
    return c == '=' ? 0 : c == 'A' ? 1 : c == 'C' ? 2 : c == 'G' ? 4 : c == 'T' ? 8 : 15;
}

// window index of IndelKey(pos, type, del, <ins_len read bases from read offset ro | the single char mm>), or SX_NO_KEY
K7A_HD uint16_t k7a_find(const k7a_view& v, const uint32_t k0, const uint32_t n_win, const int32_t pos, const unsigned type, const uint32_t del, const uint32_t ins_len,
                         const uint64_t read_byte, const uint32_t ro, const char mm)
{
    const sx_indel_key* win(v.b.keys + k0);
    uint32_t lo(0), hi(n_win);
    while (lo < hi)
    {
        const uint32_t mid((lo + hi) / 2);
        if (win[mid].pos < pos) lo = mid + 1;
        else hi = mid;
    }
    for (uint32_t k = lo; k < n_win && win[k].pos == pos; ++k)
    {
        if (win[k].type != type || win[k].del_len != del || win[k].ins_len != ins_len) continue;
        const char* seq(v.key_ins + v.key_ins_off[k0 + k]);
        bool same(true);
        for (uint32_t x = 0; x < ins_len && same; ++x) same = (seq[x] == (type == SX_INDEL_TYPE_MISMATCH ? mm : k7a_char(k7a_code(v.seq4, read_byte, ro + x))));
        if (same) return (uint16_t)k;
    }
    return SX_NO_KEY;
}

K7A_HD void k7a_add(uint16_t* keys, uint32_t& n, const uint16_t w) // std::set insert; a full array turns the surplus into SX_NO_KEY
{
    uint32_t j(0);
    while (j < n && keys[j] < w) ++j;
    if (j < n && keys[j] == w) return;
    if (n >= K7A_MAX_KEYS)
    {
        keys[K7A_MAX_KEYS - 1] = SX_NO_KEY;
        return;
    }
    for (uint32_t i = n; i > j; --i) keys[i] = keys[i - 1];
    keys[j] = w;
    ++n;
}

// keys[K7A_MAX_KEYS] <- the read's window indices (ascending, SX_NO_KEY last); returns their number
K7A_HD uint32_t k7a_read(const k7a_view& v, const uint32_t region, const uint32_t r, const uint64_t read_byte, uint16_t* keys, uint16_t& lead, uint16_t& trail)
{
    const sx_region g(v.regions[region]);
    const uint32_t k0(v.b.region_key_off[region]), n_win(v.b.region_key_off[region + 1] - k0);
    const uint32_t s0(v.b.in_seg_off[r]), aps(v.b.in_seg_off[r + 1] - s0);
    const sx_aln_seg* path(v.b.in_segs + s0);
    uint32_t first(aps), last(aps); // get_match_edge_segments
    for (uint32_t i = 0; i < aps; ++i)
    {
        const unsigned t(path[i].kind);
        if (t == SX_AP_MATCH || t == SX_AP_SEQ_MATCH || t == SX_AP_SEQ_MISMATCH)
        {
            if (first == aps) first = i;
            last = i;
        }
    }
    uint32_t n(0), ro(0);
    int32_t ref_pos(v.b.in_pos[r]);
    lead = trail = SX_NO_KEY;
    if (v.b.gate && !(v.b.gate[r] & SX_GATE_REALIGN)) return 0; // the read does not go into the search (K7g)
    bool hasLead(false), hasTrail(false);
    uint32_t i(0);
    while (i < aps)
    {
        const unsigned t(path[i].kind);
        const uint32_t len(path[i].len);
        uint32_t j(i + 1);
        const bool edge(i < first || i > last);
        // is_segment_swap_start (align_path.cpp:868-895): a run of adjacent insert / delete segments holding both kinds
        uint32_t insLen(0), delLen(0), q(i);
        for (; q < aps && (path[q].kind == SX_AP_INSERT || path[q].kind == SX_AP_DELETE); ++q) (path[q].kind == SX_AP_INSERT ? insLen : delLen) += path[q].len;
        const bool swap(insLen && delLen);
        if (edge)
        {
            if (t == SX_AP_INSERT || t == SX_AP_DELETE) // ignore all edge segments except INSERT / DELETE (:89-104); the key is the edge key
            {
                const uint16_t w(k7a_find(v, k0, n_win, ref_pos, SX_INDEL_TYPE_INDEL, t == SX_AP_DELETE ? len : 0, t == SX_AP_INSERT ? len : 0, read_byte, ro, 0));
                // getCandidateAlignment (:1495-1518) sets the edge key anew for every edge insert / delete segment -- the last one wins --
                // and getAlignmentIndels inserts that final key (:94-103), once
                if (i < first)
                {
                    lead = w;
                    hasLead = true;
                }
                else
                {
                    trail = w;
                    hasTrail = true;
                }
            }
        }
        else if (swap)
        {
            j = q;
            const uint32_t m(insLen > delLen ? insLen : delLen);
            k7a_add(keys, n, m <= v.b.opts.max_indel_size ? k7a_find(v, k0, n_win, ref_pos, SX_INDEL_TYPE_INDEL, delLen, insLen, read_byte, ro, 0) : (uint16_t)SX_NO_KEY);
        }
        else if (t == SX_AP_INSERT || t == SX_AP_DELETE)
        {
            k7a_add(keys, n,
                    len <= v.b.opts.max_indel_size ? k7a_find(v, k0, n_win, ref_pos, SX_INDEL_TYPE_INDEL, t == SX_AP_DELETE ? len : 0, t == SX_AP_INSERT ? len : 0, read_byte, ro, 0)
                                                   : (uint16_t)SX_NO_KEY); // (a breakend pair in the reference: not part of this build)
        }
        else if (t == SX_AP_MATCH || t == SX_AP_SEQ_MATCH || t == SX_AP_SEQ_MISMATCH)
        {
            for (uint32_t x = 0; x < len; ++x)
            {
                const uint8_t sbase(k7a_code(v.seq4, read_byte, ro + x));
                if (sbase == 0 || sbase == 15) continue;
                const int32_t rp(ref_pos + (int32_t)x);
                if (sbase == k7a_ref_code(v, g, rp)) continue;
                const uint16_t w(k7a_find(v, k0, n_win, rp, SX_INDEL_TYPE_MISMATCH, 1, 1, read_byte, 0, k7a_char(sbase)));
                if (w != SX_NO_KEY) k7a_add(keys, n, w); // a mismatch that is no window entry is dropped (starling_read_align.cpp:1865)
            }
        }
        for (uint32_t s = i; s < j; ++s) // increment_path
        {
            const unsigned k(path[s].kind);
            if (k == SX_AP_MATCH || k == SX_AP_INSERT || k == SX_AP_SOFT_CLIP || k == SX_AP_SEQ_MATCH || k == SX_AP_SEQ_MISMATCH) ro += path[s].len;
            if (k == SX_AP_MATCH || k == SX_AP_DELETE || k == SX_AP_SKIP || k == SX_AP_SEQ_MATCH || k == SX_AP_SEQ_MISMATCH) ref_pos += (int32_t)path[s].len;
        }
        i = j;
    }
    if (hasLead) k7a_add(keys, n, lead);
    if (hasTrail) k7a_add(keys, n, trail);
    return n;
}

// ---------------------------------------------------------------------------------------------------------------------------
// K7g realign_gates: the front of realignAndScoreRead (starling_read_align.cpp:2045-2062), one read
// ---------------------------------------------------------------------------------------------------------------------------
#define K7G_MAX_SEGS 64u // path segments of a mapper alignment handled here (longer: the read is left to the caller, gate 0)

K7A_HD bool k7g_align_match(const unsigned t) { return t == SX_AP_MATCH || t == SX_AP_SEQ_MATCH || t == SX_AP_SEQ_MISMATCH; }
K7A_HD bool k7g_read_kind(const unsigned t) { return k7g_align_match(t) || t == SX_AP_INSERT || t == SX_AP_SOFT_CLIP; }
K7A_HD bool k7g_ref_kind(const unsigned t) { return k7g_align_match(t) || t == SX_AP_DELETE || t == SX_AP_SKIP; }

K7A_HD void k7g_ends(const sx_aln_seg* p, const uint32_t n, uint32_t& first, uint32_t& last) // get_match_edge_segments, align_path.cpp:736-752
{
    first = last = n;
    for (uint32_t i = 0; i < n; ++i)
        if (k7g_align_match(p[i].kind))
        {
            if (first == n) first = i;
            last = i;
        }
}

// appends ps to out[0 .. n) as matchify_edge_segment_type does (alignment_util.cpp:128-175): a segment that becomes a match (`to_match`)
// extends a match before it
K7A_HD void k7g_put(sx_aln_seg* out, uint32_t& n, const sx_aln_seg ps, const bool to_match)
{
    if (to_match && n > 0 && out[n - 1].kind == SX_AP_MATCH) out[n - 1].len = (uint16_t)(out[n - 1].len + ps.len);
    else out[n++] = sx_aln_seg{ps.len, (uint8_t)(to_match ? SX_AP_MATCH : ps.kind), 0};
}

// returns gate bits; out_pos / out_segs[0 .. n_slots) receive the normalized alignment (+ zero-length HARD_CLIP pads).  The tests take the
// mapper's alignment as it is; only edge-indel removal and the soft-clip matchify rewrite it, straight into out_segs.
K7A_HD uint32_t k7g_read(const sx_gate_batch& b, const uint32_t region, const uint32_t r, int32_t& out_pos, sx_aln_seg* out_segs)
{
    const uint32_t s0(b.seg_off[r]), n_slots(b.seg_off[r + 1] - s0);
    const sx_aln_seg* al(b.raw_segs + s0);
    const int32_t al_pos(b.raw_pos[r]);
    out_pos = al_pos;
    for (uint32_t i = 0; i < n_slots; ++i) out_segs[i] = al[i];
    if (n_slots == 0 || n_slots > K7G_MAX_SEGS) return 0;
    // ---- is_realignable = !is_overmax, alignment.cpp:34-50
    for (uint32_t i = 1; i + 1 < n_slots; ++i)
        if ((al[i].kind == SX_AP_INSERT || al[i].kind == SX_AP_DELETE) && al[i].len > b.max_indel_size) return 0;
    // ---- check_for_candidate_indel_overlap, :222-283
    {
        uint32_t lead(0), trail(0), asize(0);
        for (uint32_t i = 0; i < n_slots; ++i) // unalignedPrefixSize
        {
            const unsigned t(al[i].kind);
            if (!(t == SX_AP_INSERT || t == SX_AP_HARD_CLIP || t == SX_AP_SOFT_CLIP)) break;
            if (k7g_read_kind(t)) lead += al[i].len;
        }
        for (uint32_t i = n_slots; i-- > 0;) // unalignedSuffixSize
        {
            const unsigned t(al[i].kind);
            if (!(t == SX_AP_INSERT || t == SX_AP_HARD_CLIP || t == SX_AP_SOFT_CLIP)) break;
            if (k7g_read_kind(t)) trail += al[i].len;
        }
        for (uint32_t i = 0; i < n_slots; ++i)
            if (k7g_ref_kind(al[i].kind)) asize += al[i].len;
        const int32_t pb(al_pos - (int32_t)lead), pe(al_pos + (int32_t)asize + (int32_t)trail), len((int32_t)b.read_len[r]);
        int32_t zb(pb < pe - len ? pb : pe - len);
        zb = zb > 0 ? zb : 0;
        const int32_t ze(pe > pb + len ? pe : pb + len);
        if (!(zb >= b.realign_begin[region] && ze <= b.realign_end[region])) return 0;
        const uint32_t k0(b.region_key_off[region]), n_win(b.region_key_off[region + 1] - k0);
        const sx_indel_key* win(b.keys + k0);
        uint32_t k(0);
        while (k < n_win && (int64_t)win[k].pos < (int64_t)zb - (int64_t)b.max_indel_size) ++k; // rangeIterator(zb, ze), IndelBuffer.cpp:76-91
        while (k < n_win && win[k].pos < ze && win[k].pos + (int32_t)win[k].del_len < zb) ++k;
        bool overlap(false);
        for (; k < n_win && win[k].pos < ze && !overlap; ++k)
        {
            const sx_indel_key& ik(win[k]);
            bool hit;
            if (ik.type == SX_INDEL_TYPE_MISMATCH) hit = (ik.pos >= zb && ik.pos < ze);
            else
            {
                const int32_t rp(ik.pos + (int32_t)ik.del_len);
                hit = (ik.pos > zb && ik.pos < ze) || (rp != ik.pos && rp > zb && rp < ze);
            }
            if (hit && (ik.flags & SX_IKF_CANDIDATE)) overlap = true;
        }
        if (!overlap) return 0;
    }
    // ---- normalizeInputAlignmentIndels, :2000-2021: remove_edge_deletions (alignment_util.cpp:89-123) and matchify_edge_insertions, one pass
    const unsigned pins(b.pin_flags ? b.pin_flags[r] : 0u);
    const bool rm_lead(!(pins & 1u)), rm_trail(!(pins & 2u));
    uint32_t first, last;
    k7g_ends(al, n_slots, first, last);
    bool edge(false); // is_edge_readref_len_segment, align_path.cpp:827-846
    if (rm_lead || rm_trail)
        for (uint32_t i = 0; i < n_slots; ++i)
        {
            const unsigned t(al[i].kind);
            if ((i < first || i > last) && (t == SX_AP_INSERT || t == SX_AP_DELETE || t == SX_AP_SKIP || t == SX_AP_SOFT_CLIP)) edge = true;
        }
    int32_t pos(al_pos);
    uint32_t n(0);
    bool soft(false);
    for (uint32_t i = 0; i < n_slots; ++i)
    {
        const sx_aln_seg ps(al[i]);
        const bool is_lead(i < first), is_trail(i > last), rm((is_lead && rm_lead) || (is_trail && rm_trail));
        soft = soft || ps.kind == SX_AP_SOFT_CLIP;
        if (!edge) out_segs[n++] = sx_aln_seg{ps.len, ps.kind, 0};
        else if (ps.kind == SX_AP_DELETE && rm) // an edge deletion goes
        {
            if (is_lead) pos += (int32_t)ps.len;
        }
        else // an edge insertion becomes a match (the deletions' removal leaves every other segment on its side of the matches)
        {
            const bool target(rm && ps.kind == SX_AP_INSERT);
            if (target && is_lead) pos -= (int32_t)ps.len;
            k7g_put(out_segs, n, ps, target || k7g_align_match(ps.kind));
        }
    }
    // ---- soft clips become matches, :2051-2057: matchify_edge_soft_clip of the path above, in place (it never grows)
    uint32_t gate(SX_GATE_REALIGN);
    if (soft)
    {
        gate |= SX_GATE_SOFT_CLIPPED;
        k7g_ends(out_segs, n, first, last);
        const uint32_t m(n);
        n = 0;
        for (uint32_t i = 0; i < m; ++i)
        {
            const sx_aln_seg ps(out_segs[i]);
            const bool target((i < first || i > last) && ps.kind == SX_AP_SOFT_CLIP);
            if (target && i < first) pos -= (int32_t)ps.len;
            k7g_put(out_segs, n, ps, target || k7g_align_match(ps.kind));
        }
    }
    if (pos < 0) // :2062 -- the read keeps its mapper's alignment
    {
        for (uint32_t i = 0; i < n_slots; ++i) out_segs[i] = al[i];
        return gate & ~SX_GATE_REALIGN;
    }
    out_pos = pos;
    for (uint32_t i = n; i < n_slots; ++i) out_segs[i] = sx_aln_seg{0, SX_AP_HARD_CLIP, 0};
    return gate;
}
