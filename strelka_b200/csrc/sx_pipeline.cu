// sx_pipeline.cu -- sx_process_window_dev: the READ_BUFFER and POST_ALIGN stages of the reference's position processor for a window of
// positions as ONE device-resident pass (include/strelka_b200.h, "process_window"):
//
//   align_pos          /root/reference/src/c++/lib/starling_common/starling_pos_processor_base.cpp:732-773
//   pileup_pos_reads   :1107-1123 (pileup_read_segment :1127-1421)
//   computeSampleDiploidSiteGenotype   applications/starling/starling_pos_processor.cpp:254-267
//
// Nothing here is a new algorithm: the function owns the buffers between the stages and enqueues the stage launchers (each beside its
// kernels: sx_k7g_run ... sx_k2a_run) on the context's compute stream.  What crosses to the host between the stages is the handful of totals
// that size the next stage's buffers and launch; every array stays in HBM.  Small kernels of its own prepare what no stage produces: the
// read index of sx_read_index.cu (per-read regions and byte offsets, which K7g, K7a, K7b and K9 read) and the per-read facts read off it --
// 'N' counts, buffer positions, pin bits -- with the window entries' longest insert (prep), the sub-mapped reads' gate (align_pos :746),
// and K4's read records from K9's best alignments (pileup_read_segment's preamble :1136-1171).
#include "sx_internal.h"
#include "sx_read_index.cuh"

#include <algorithm>
#include <cstring>

namespace
{
struct prep_out
{
    uint32_t* region;    // [n_reads] the read's region (this and the two offsets: the read index, sx_read_index.cu)
    uint32_t* seq_off;   // [n_reads + 1] byte offset of its packed bases (reads of a region back to back, each on a byte boundary),
    uint32_t* qual_off;  // [n_reads + 1] ... of its qualities (qual_bits 4: packed like the bases; else one byte per base),
    int32_t* bpos;       // [n_reads] rseg.buffer_pos,
    uint16_t* non_ambig; // [n_reads] bases that are not 'N',
    uint8_t* pin;        // [n_reads] bit 0 / 1: edge pins
    uint32_t* maxima;    // [4] max insert length of a window entry, max |best pos - buffer pos|, max reference span, (unused)
};

// the per-read facts only the window pass reads, from the read index's offsets: 'N' counts (K6), buffer positions (K4), pin bits (K7g, K9)
__global__ void sxp_read_facts_kernel(const sx_window_batch b, const prep_out o)
{
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < b.n_reads; r += gridDim.x * blockDim.x)
    {
        const uint32_t len(b.read_len[r]);
        o.non_ambig[r] = (uint16_t)(len - sxi_count_n(b.seq4 + o.seq_off[r], len)); // score_indels :866-875
        const uint32_t s0(b.raw_seg_off[r]);
        o.bpos[r] = sxi_buffer_pos(b.raw_pos[r], b.raw_segs + s0, b.raw_seg_off[r + 1] - s0);
        const unsigned f(b.read_flags[r]);
        o.pin[r] = (uint8_t)(((f & SX_PRF_PIN_FIRST) ? 1u : 0u) | ((f & SX_PRF_PIN_SECOND) ? 2u : 0u));
    }
}

// the longest insert of a window entry (sizes K7b's insert pool)
__global__ void sxp_key_max_kernel(const uint32_t n_keys, const sx_indel_key* __restrict__ keys, uint32_t* __restrict__ maxima)
{
    uint32_t m(0);
    for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n_keys; k += gridDim.x * blockDim.x) m = max(m, (uint32_t)keys[k].ins_len);
    if (m) atomicMax(&maxima[0], m);
}

// align_pos :746: only tier1 / tier2 mappings are realigned
__global__ void sxp_submapped_gate_kernel(const uint32_t n, const uint8_t* __restrict__ flags, uint8_t* __restrict__ gate)
{
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x)
        if (!(flags[r] & SX_PRF_TIER1OR2)) gate[r] = 0;
}

// K4's read records from K9's best alignments (+ the preamble of pileup_read_segment that needs the mapper's alignment: a read that was
// not realigned and whose every indel exceeds maxIndelSize is not piled up, :1145-1148 is_any_nonovermax)
__global__ void sxp_pileup_reads_kernel(const sx_window_batch b, const prep_out p, const int32_t* __restrict__ best_pos, const uint32_t* __restrict__ best_seg_off,
                                        const sx_aln_seg* __restrict__ best_segs, const uint8_t* __restrict__ realign_status, sx_pileup_read* __restrict__ out)
{
    uint32_t max_shift(0), max_span(0);
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r <= b.n_reads; r += gridDim.x * blockDim.x)
    {
        sx_pileup_read rd;
        rd.seq_off = p.seq_off[r];
        rd.qual_off = p.qual_off[r];
        rd.seg_off = best_seg_off[r];
        rd.pos = 0;
        rd.len = 0;
        rd.mapq = 0;
        rd.flags = 0;
        if (r < b.n_reads)
        {
            rd.pos = best_pos[r];
            rd.len = b.read_len[r];
            rd.mapq = b.mapq[r];
            unsigned f(b.read_flags[r] & (SX_PRF_FWD | SX_PRF_TIER1 | SX_PRF_TIER1OR2 | SX_PRF_PIN_FIRST | SX_PRF_PIN_SECOND));
            if (!(realign_status[r] & SX_REALIGN_ST_REALIGNED))
            {
                // alignment::is_overmax (alignment.cpp:34-50) of the only alignment the read has
                bool overmax(false);
                const uint32_t s0(b.raw_seg_off[r]), s1(b.raw_seg_off[r + 1]);
                for (uint32_t s = s0 + 1; s + 1 < s1; ++s)
                    if ((b.raw_segs[s].kind == SX_AP_INSERT || b.raw_segs[s].kind == SX_AP_DELETE) && b.raw_segs[s].len > b.enum_opts.max_indel_size) overmax = true;
                if (overmax) f |= SX_PRF_SKIP;
            }
            rd.flags = (uint8_t)f;
            uint32_t span(0);
            for (uint32_t s = best_seg_off[r]; s < best_seg_off[r + 1]; ++s)
            {
                const unsigned k(best_segs[s].kind);
                if (k == SX_SEG_MATCH || k == SX_SEG_DELETE || k == SX_SEG_SKIP) span += best_segs[s].len;
            }
            const int32_t d(rd.pos - p.bpos[r]);
            max_shift = max(max_shift, (uint32_t)(d < 0 ? -d : d));
            max_span = max(max_span, span);
        }
        out[r] = rd;
    }
    if (max_shift) atomicMax(&p.maxima[1], max_shift);
    if (max_span) atomicMax(&p.maxima[2], max_span);
}

// ---- order-preserving compaction of the items a selector keeps: per 1024-item chunk a count, an exclusive scan over the chunks (sx_scan), ranked
// writes.  A selector S has `bool keep(i)` and `S::record make(i)` (the record of a kept item); one instance per record kind.
constexpr uint32_t VC_CHUNK = 1024, VC_THREADS = 256;

template <class S> __global__ void __launch_bounds__(VC_THREADS) sxp_compact_count_kernel(const S sel, const uint32_t n, uint32_t* __restrict__ chunk_cnt)
{
    const uint32_t base(blockIdx.x * VC_CHUNK);
    int total(0);
    for (uint32_t i = 0; i < VC_CHUNK / VC_THREADS; ++i)
    {
        const uint32_t s(base + i * VC_THREADS + threadIdx.x);
        total += __syncthreads_count(s < n && sel.keep(s));
    }
    if (threadIdx.x == 0) chunk_cnt[blockIdx.x] = (uint32_t)total;
}

template <class S>
__global__ void __launch_bounds__(VC_THREADS) sxp_compact_write_kernel(const S sel, const uint32_t n, const uint32_t* __restrict__ chunk_off, typename S::record* __restrict__ out,
                                                                       const uint32_t cap)
{
    __shared__ uint32_t warp_cnt[VC_THREADS / 32];
    __shared__ uint32_t run;
    if (threadIdx.x == 0) run = chunk_off[blockIdx.x];
    __syncthreads();
    const uint32_t base(blockIdx.x * VC_CHUNK), lane(threadIdx.x & 31), wid(threadIdx.x >> 5);
    for (uint32_t i = 0; i < VC_CHUNK / VC_THREADS; ++i)
    {
        const uint32_t s(base + i * VC_THREADS + threadIdx.x);
        const bool v(s < n && sel.keep(s));
        const unsigned m(__ballot_sync(0xffffffffu, v));
        if (lane == 0) warp_cnt[wid] = __popc(m);
        __syncthreads();
        uint32_t before(run);
        for (uint32_t k = 0; k < wid; ++k) before += warp_cnt[k];
        if (v)
        {
            const uint32_t at(before + __popc(m & ((1u << lane) - 1u)));
            if (at < cap) out[at] = sel.make(s);
        }
        __syncthreads();
        if (threadIdx.x == 0)
        {
            uint32_t t(0);
            for (uint32_t k = 0; k < VC_THREADS / 32; ++k) t += warp_cnt[k];
            run += t;
        }
        __syncthreads();
    }
}

// germline: the computed sites whose most likely genotype is not the reference's
struct variant_site_sel
{
    using record = sx_site_call;
    const sx_digt_result* gl;
    const uint32_t* site_off;
    int32_t report_begin;
    __device__ bool keep(const uint32_t s) const { return gl[s].is_computed && gl[s].genome.max_gt != gl[s].ref_gt; }
    __device__ record make(const uint32_t s) const
    {
        sx_site_call c;
        c.pos = report_begin + (int32_t)s;
        c.n_calls = site_off[s + 1] - site_off[s];
        c.gl = gl[s];
        return c;
    }
};

// somatic SNV: somatic_snv_genotype_grid::is_output() (somatic_result_set.hh:62-71).  qphred is defined where the model ran; a forced position
// whose reference base is 'N' loses the flag (position_somatic_snv_strand_grid.cpp:242-246).
struct somatic_site_sel
{
    using record = sx_somatic_site_call;
    const sx_ssnv_result* r;
    const uint8_t* forced; // or NULL
    const char* ref_base;
    const uint32_t* n_off;
    const uint32_t* t_off;
    int32_t report_begin;
    __device__ bool keep(const uint32_t s) const { return (r[s].is_computed && r[s].qphred != 0) || (forced && forced[s] && ref_base[s] != 'N'); }
    __device__ record make(const uint32_t s) const
    {
        sx_somatic_site_call c;
        c.pos = report_begin + (int32_t)s;
        c.n_calls[0] = n_off[s + 1] - n_off[s];
        c.n_calls[1] = t_off[s + 1] - t_off[s];
        c.pad = 0;
        c.r = r[s];
        return c;
    }
};

// somatic indel: a locus the link flagged (the caller's CPU path calls it), else somatic_indel_call::is_output() (somatic_result_set.hh:86-96)
// of a locus that process_pos_indel_somatic calls at all -- an unforced candidate with both read_path_lnp empty is skipped
// (strelka_pos_processor.cpp:324-327).  The link's read_off holds the offsets of the two lists of locus l at 2l, 2l+1, 2l+2.
struct somatic_indel_sel
{
    using record = sx_somatic_indel_call;
    const sx_sindel_result* r;
    const uint8_t* forced;
    const uint32_t* status;
    const uint32_t* read_off;
    __device__ bool keep(const uint32_t l) const
    {
        if (status[l] || forced[l]) return true;
        return r[l].qphred != 0 && read_off[2 * l + 2] != read_off[2 * l];
    }
    __device__ record make(const uint32_t l) const
    {
        sx_somatic_indel_call c;
        c.locus = l;
        c.pad = 0;
        c.r = r[l];
        return c;
    }
};

// the window pass's buffers: `count` elements and 64 bytes of slack
template <typename T> int take(sx_ctx* ctx, sx_slot slot, size_t count, T*& p) { return sx_take(ctx, slot, count, p, 64); }

// the caller's array, or the context's own buffer when the caller passed NULL
template <typename T> int pick(sx_ctx* ctx, sx_slot slot, size_t count, T* user, T*& p)
{
    if (user)
    {
        p = user;
        return SX_OK;
    }
    return take(ctx, slot, count, p);
}

int read_status(sx_ctx* ctx, int* st)
{
    SX_CUDA(ctx, cudaMemcpyAsync(st, ctx->d_status, sizeof(int), cudaMemcpyDeviceToHost, ctx->s_compute));
    return SX_OK;
}

// The compaction of `n` items (n > 0) into out[cap]: two launches and the scan's, on the compute stream; *total (host memory) receives the
// number of kept items once the stream has passed the copy.
template <class S> int compact(sx_ctx* ctx, const S& sel, const uint32_t n, sx_slot chunk_slot, sx_slot sums_slot, typename S::record* out, const uint32_t cap,
                               uint32_t* total, unsigned* launches)
{
    cudaStream_t st(ctx->s_compute);
    const uint32_t n_chunks((n + VC_CHUNK - 1) / VC_CHUNK);
    uint32_t* chunk_cnt(nullptr);
    int rc;
    if ((rc = take(ctx, chunk_slot, (size_t)n_chunks + 4, chunk_cnt))) return rc;
    sxp_compact_count_kernel<<<n_chunks, VC_THREADS, 0, st>>>(sel, n, chunk_cnt);
    SX_CUDA(ctx, cudaGetLastError());
    const sx_scan_set J = {1, {{chunk_cnt, n_chunks, SX_SCAN_EXCLUSIVE | SX_SCAN_CLOSE, nullptr}}};
    if ((rc = sx_scan(ctx, sums_slot, J, launches))) return rc;
    sxp_compact_write_kernel<<<n_chunks, VC_THREADS, 0, st>>>(sel, n, chunk_cnt, out, cap);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 2;
    SX_CUDA(ctx, cudaMemcpyAsync(total, chunk_cnt + n_chunks, 4, cudaMemcpyDeviceToHost, st));
    return SX_OK;
}

// The slots of the window pass's results that a later stage reads, where the caller's output array does not take their place: the pass's own
// (WIN_SLOTS), or a bank that survives a second pass on the same context (the somatic pass's normal sample)
// t2_all_bases: the tier2 columns' own buffer is sized like the tier1 columns' (no more calls than the reads have bases) also without tier2
// evidence -- the pile-up puts the tier2 reads' calls there either way, and the somatic pass reads the columns of both samples from these
// buffers.  (The germline pass keeps its 64-call buffer.)
struct win_slots
{
    sx_slot non_ambig, recs, n_rec, site_off, t2_off, calls, t2_calls;
    bool t2_all_bases;
};
constexpr win_slots WIN_SLOTS = {SX_SLOT_WIN_NON_AMBIG, SX_SLOT_WIN_RECS, SX_SLOT_WIN_N_REC, SX_SLOT_WIN_SITE_OFF, SX_SLOT_WIN_T2_OFF, SX_SLOT_WIN_CALLS, SX_SLOT_WIN_T2_CALLS, false};
constexpr win_slots SWIN_TUMOR_SLOTS = {SX_SLOT_WIN_NON_AMBIG, SX_SLOT_WIN_RECS, SX_SLOT_WIN_N_REC, SX_SLOT_WIN_SITE_OFF, SX_SLOT_WIN_T2_OFF, SX_SLOT_WIN_CALLS,
                                        SX_SLOT_WIN_T2_CALLS, true};
constexpr win_slots SWIN_NORMAL_SLOTS = {SX_SLOT_SWIN_NON_AMBIG, SX_SLOT_SWIN_RECS, SX_SLOT_SWIN_N_REC, SX_SLOT_SWIN_SITE_OFF, SX_SLOT_SWIN_T2_OFF, SX_SLOT_SWIN_CALLS,
                                         SX_SLOT_SWIN_T2_CALLS, true};

// ... and where those results are once the pass has run
struct win_kept
{
    const uint16_t* non_ambig;
    const sx_read_indel_score* recs;
    const uint32_t* n_rec;
    sx_pileup_columns cols;
};
} // namespace

extern "C" void sx_default_window_opts(sx_window_batch* b)
{
    if (!b) return;
    sx_default_enum_opts(&b->enum_opts);
    b->enum_opts.max_alns_per_read = 5000; // opt.max_realignment_candidates (starling_base_shared.hh:160): no read is left to the caller for its alignment count
    sx_default_score_indels_opts(&b->score_opts);
    sx_default_pileup_opts(&b->pileup_opts);
    b->is_always_test = 1;
    b->do_site_gl = 1;
    b->is_retain_optimal_soft_clipping = 0;
    b->reserved_ = 0;
}

extern "C" int sx_last_window_timing(const sx_ctx* ctx, float* ms)
{
    if (!ctx || !ms) return SX_ERR_ARG;
    for (int i = 0; i < SX_WIN_N_STAGES; ++i) ms[i] = ctx->win_ms[i];
    return SX_OK;
}

namespace
{
// the window pass of sx_process_window_dev, which sx_process_window runs on the window it has uploaded
// metrics: K4m on the pass's own pile-up batch after the last stage (sx_process_window_metrics_dev), NULL: not run
struct win_metrics
{
    const sx_pileup_metrics_opts* opts;
    sx_pileup_metrics_rec* out;
};
int window_pass(sx_ctx* ctx, const sx_window_batch* b, sx_window_out* out, uint32_t* totals_host, const win_slots& S = WIN_SLOTS, win_kept* kept = nullptr,
                const win_metrics& M = win_metrics{nullptr, nullptr})
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    if (!b || !out) return sx_fail(ctx, SX_ERR_ARG, "sx_process_window_dev: NULL argument");
    if (b->report_end < b->report_begin) return sx_fail(ctx, SX_ERR_ARG, "sx_process_window_dev: empty report range");
    if (b->n_reads && (!b->region_read_off || !b->region_key_off || !b->realign_begin || !b->realign_end || !b->raw_pos || !b->raw_seg_off || !b->raw_segs ||
                       !b->read_len || !b->read_flags || !b->mapq || !b->use_key_off || !b->rec_off || !b->regions || !b->seq4 || !b->qual || !b->ref ||
                       (b->n_keys && (!b->keys || !b->key_ins_off || !b->key_ins)) || b->n_regions == 0))
        return sx_fail(ctx, SX_ERR_ARG, "sx_process_window_dev: NULL array");
    if (b->qual_bits != 0 && b->qual_bits != 8 && b->qual_bits != 4) return sx_fail(ctx, SX_ERR_ARG, "sx_process_window_dev: qual_bits must be 0, 8 or 4");
    if (b->is_retain_optimal_soft_clipping)
        return sx_fail(ctx, SX_ERR_UNSUPPORTED, "sx_process_window_dev: isRetainOptimalSoftClipping (the RNA workflow's soft-clip retention test) is outside the accelerated path");
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st(ctx->s_compute);
    for (int i = 0; i <= SX_WIN_N_STAGES + (M.out ? 1 : 0); ++i)
        if (!ctx->ev_win[i]) SX_CUDA(ctx, cudaEventCreate(&ctx->ev_win[i]));
    const uint32_t n(b->n_reads), nr(b->n_regions);
    const uint32_t n_sites((uint32_t)(b->report_end - b->report_begin));
    unsigned launches(0);
    int rc;
    uint32_t totals[SX_WIN_TOTALS] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    const int cap_grid(ctx->sm_count * 16);
    const auto grid = [cap_grid](const uint32_t m) { return (unsigned)std::max(1, std::min<int>((int)((m + 127) / 128), cap_grid)); };
    auto mark = [&](int i) { return cudaEventRecord(ctx->ev_win[i], st); };

    // ---------------------------------------------------------------------------------------------------------------- prep
    SX_CUDA(ctx, mark(SX_WIN_ST_PREP));
    prep_out P;
    if ((rc = take(ctx, SX_SLOT_WIN_READ_REGION, (size_t)n + 1, P.region))) return rc;
    if ((rc = take(ctx, SX_SLOT_WIN_SEQ_OFF, (size_t)n + 1, P.seq_off))) return rc;
    if ((rc = take(ctx, SX_SLOT_WIN_QUAL_OFF, (size_t)n + 1, P.qual_off))) return rc;
    if ((rc = take(ctx, SX_SLOT_WIN_BPOS, (size_t)n + 1, P.bpos))) return rc;
    if ((rc = take(ctx, S.non_ambig, (size_t)n + 1, P.non_ambig))) return rc;
    if ((rc = take(ctx, SX_SLOT_WIN_PIN, (size_t)n + 1, P.pin))) return rc;
    if ((rc = take(ctx, SX_SLOT_WIN_MAXIMA, 4, P.maxima))) return rc;
    SX_CUDA(ctx, cudaMemsetAsync(P.maxima, 0, 16, st));
    uint32_t n_raw_segs(0);
    if (n)
    {
        sx_read_index_in in;
        memset(&in, 0, sizeof(in));
        in.n_regions = nr;
        in.n_reads = n;
        in.qual_bits = b->qual_bits;
        in.region_read_off = b->region_read_off;
        in.read_len = b->read_len;
        in.regions = b->regions;
        const sx_read_index ix = {P.region, P.seq_off, P.qual_off};
        if ((rc = sx_read_index_run(ctx, &in, &ix, &launches))) return rc;
        sxp_read_facts_kernel<<<grid(n), 128, 0, st>>>(*b, P);
        SX_CUDA(ctx, cudaGetLastError());
        sxp_key_max_kernel<<<grid(b->n_keys), 128, 0, st>>>(b->n_keys, b->keys, P.maxima);
        SX_CUDA(ctx, cudaGetLastError());
        launches += 2;
        SX_CUDA(ctx, cudaMemcpyAsync(&n_raw_segs, b->raw_seg_off + n, 4, cudaMemcpyDeviceToHost, st));
    }
    // ---------------------------------------------------------------------------------------------------------------- K7g gates
    SX_CUDA(ctx, mark(SX_WIN_ST_GATES));
    SX_CUDA(ctx, cudaStreamSynchronize(st)); // n_raw_segs sizes the normalized-alignment array
    uint8_t* gate(nullptr);
    int32_t* in_pos(nullptr);
    sx_aln_seg* in_segs(nullptr);
    if ((rc = pick(ctx, SX_SLOT_WIN_GATE, (size_t)n + 1, out->gate, gate))) return rc;
    if ((rc = take(ctx, SX_SLOT_WIN_IN_POS, (size_t)n + 1, in_pos))) return rc;
    if ((rc = take(ctx, SX_SLOT_WIN_IN_SEGS, (size_t)n_raw_segs + 1, in_segs))) return rc;
    {
        sx_gate_batch gb;
        memset(&gb, 0, sizeof(gb));
        gb.n_regions = nr;
        gb.n_reads = n;
        gb.region_read_off = b->region_read_off;
        gb.region_key_off = b->region_key_off;
        gb.keys = b->keys;
        gb.realign_begin = b->realign_begin;
        gb.realign_end = b->realign_end;
        gb.raw_pos = b->raw_pos;
        gb.seg_off = b->raw_seg_off;
        gb.raw_segs = b->raw_segs;
        gb.read_len = b->read_len;
        gb.pin_flags = P.pin;
        gb.max_indel_size = b->enum_opts.max_indel_size;
        sx_gate_out go = {gate, in_pos, in_segs};
        if ((rc = sx_k7g_run(ctx, &gb, &go, P.region, &launches))) return rc;
        if (n)
        {
            sxp_submapped_gate_kernel<<<grid(n), 128, 0, st>>>(n, b->read_flags, gate);
            SX_CUDA(ctx, cudaGetLastError());
            ++launches;
        }
    }
    // ---------------------------------------------------------------------------------------------------------------- K7a keys of the input alignments
    SX_CUDA(ctx, mark(SX_WIN_ST_KEYS));
    sx_enum_batch eb;
    memset(&eb, 0, sizeof(eb));
    eb.n_regions = nr;
    eb.n_reads = n;
    eb.n_keys = b->n_keys;
    eb.region_read_off = b->region_read_off;
    eb.region_key_off = b->region_key_off;
    eb.keys = b->keys;
    eb.key_hap = b->key_hap;
    eb.realign_begin = b->realign_begin;
    eb.realign_end = b->realign_end;
    eb.in_pos = in_pos;
    eb.in_seg_off = b->raw_seg_off;
    eb.in_segs = in_segs;
    eb.use_key_off = b->use_key_off;
    eb.use_keys = b->use_keys;
    eb.read_len = b->read_len;
    eb.gate = gate;
    eb.opts = b->enum_opts;
    sx_prep_out po;
    uint32_t* in_key_off(nullptr);
    uint16_t *in_keys(nullptr), *in_lead(nullptr), *in_trail(nullptr);
    uint32_t cap_in_keys(std::max<uint32_t>(64, 8u * n));
    if ((rc = take(ctx, SX_SLOT_WIN_KEY_TOTALS, 4, po.totals))) return rc;
    if ((rc = take(ctx, SX_SLOT_WIN_IN_KEY_OFF, (size_t)n + 1, in_key_off))) return rc;
    if ((rc = take(ctx, SX_SLOT_WIN_IN_LEAD, (size_t)n + 1, in_lead))) return rc;
    if ((rc = take(ctx, SX_SLOT_WIN_IN_TRAIL, (size_t)n + 1, in_trail))) return rc;
    uint32_t n_in_keys(0);
    for (int attempt = 0; n && attempt < 2; ++attempt)
    {
        if ((rc = take(ctx, SX_SLOT_WIN_IN_KEYS, (size_t)cap_in_keys + 1, in_keys))) return rc;
        po.cap_keys = cap_in_keys;
        po.in_key_off = in_key_off;
        po.in_keys = in_keys;
        po.in_lead_key = in_lead;
        po.in_trail_key = in_trail;
        if ((rc = sx_k7a_run(ctx, &eb, b->regions, b->seq4, b->ref, b->key_ins_off, b->key_ins, &po, P.region, P.seq_off, &launches))) return rc;
        SX_CUDA(ctx, cudaMemcpyAsync(&n_in_keys, po.totals, 4, cudaMemcpyDeviceToHost, st));
        SX_CUDA(ctx, cudaStreamSynchronize(st));
        if (n_in_keys <= cap_in_keys) break;
        if (attempt == 1) return sx_fail(ctx, SX_ERR_CAPACITY, "sx_process_window_dev: input-alignment keys (%u) exceed the retried capacity", n_in_keys);
        cap_in_keys = n_in_keys + 64; // the count pass has said what is needed: once more with that
        SX_CUDA(ctx, cudaMemsetAsync(ctx->d_status, 0, sizeof(int), st)); // (clears SX_ST_K7A_CAP)
    }
    eb.in_key_off = in_key_off;
    eb.in_keys = in_keys;
    eb.in_lead_key = in_lead;
    eb.in_trail_key = in_trail;
    // ---------------------------------------------------------------------------------------------------------------- K7 enumeration
    SX_CUDA(ctx, mark(SX_WIN_ST_ENUMERATE));
    sx_enum_out eo;
    memset(&eo, 0, sizeof(eo));
    uint8_t* enum_status(nullptr);
    if ((rc = pick(ctx, SX_SLOT_WIN_ENUM_STATUS, (size_t)n + 1, out->enum_status, enum_status))) return rc;
    if ((rc = take(ctx, SX_SLOT_WIN_ENUM_TOTALS, 4, eo.totals))) return rc;
    if ((rc = take(ctx, SX_SLOT_WIN_ALN_OFF, (size_t)n + 1, eo.aln_off))) return rc;
    eo.status = enum_status;
    uint32_t capA(std::max<uint32_t>(256, 12u * n)), capS(std::max<uint32_t>(1024, 56u * n)), capK(std::max<uint32_t>(512, 28u * n));
    uint32_t nA(0), nS(0), nK(0);
    uint32_t maxima[4] = {0, 0, 0, 0};
    for (int attempt = 0; n && attempt < 2; ++attempt)
    {
        eo.cap_alns = capA;
        eo.cap_segs = capS;
        eo.cap_keys = capK;
        if ((rc = take(ctx, SX_SLOT_WIN_ALN_POS, (size_t)capA + 1, eo.aln_pos))) return rc;
        if ((rc = take(ctx, SX_SLOT_WIN_ALN_SEG_OFF, (size_t)capA + 2, eo.aln_seg_off))) return rc;
        if ((rc = take(ctx, SX_SLOT_WIN_SEGS, (size_t)capS + 16, eo.segs))) return rc;
        if ((rc = take(ctx, SX_SLOT_WIN_ALN_KEY_OFF, (size_t)capA + 2, eo.aln_key_off))) return rc;
        if ((rc = take(ctx, SX_SLOT_WIN_ALN_KEYS, (size_t)capK + 16, eo.aln_keys))) return rc;
        if ((rc = take(ctx, SX_SLOT_WIN_ALN_LEAD, (size_t)capA + 1, eo.aln_lead_key))) return rc;
        if ((rc = take(ctx, SX_SLOT_WIN_ALN_TRAIL, (size_t)capA + 1, eo.aln_trail_key))) return rc;
        if ((rc = sx_k7_run(ctx, &eb, &eo, &launches))) return rc;
        uint32_t t3[3] = {0, 0, 0};
        SX_CUDA(ctx, cudaMemcpyAsync(t3, eo.totals, 12, cudaMemcpyDeviceToHost, st));
        SX_CUDA(ctx, cudaMemcpyAsync(maxima, P.maxima, 16, cudaMemcpyDeviceToHost, st));
        SX_CUDA(ctx, cudaStreamSynchronize(st));
        nA = t3[0];
        nS = t3[1];
        nK = t3[2];
        if (nA <= capA && nS <= capS && nK <= capK) break;
        if (attempt == 1) return sx_fail(ctx, SX_ERR_CAPACITY, "sx_process_window_dev: the enumeration (%u alignments, %u segments, %u keys) exceeds the retried capacity", nA, nS, nK);
        capA = std::max(capA, nA + 64); // the search has said what it produces: once more with that
        capS = std::max(capS, nS + 64);
        capK = std::max(capK, nK + 64);
        SX_CUDA(ctx, cudaMemsetAsync(ctx->d_status, 0, sizeof(int), st)); // (clears SX_ST_K7_CAP)
    }
    totals[0] = nA;
    totals[1] = nS;
    totals[2] = nK;
    // ---------------------------------------------------------------------------------------------------------------- K7b link
    SX_CUDA(ctx, mark(SX_WIN_ST_LINK));
    sx_link_out lo;
    memset(&lo, 0, sizeof(lo));
    const uint32_t max_ins(std::max<uint32_t>(1, maxima[0]));
    lo.cap_segs = 2u * nS + 8u * nr + 64u;
    {
        const unsigned long long want((unsigned long long)nS * max_ins + 16ull * nr + 64ull);
        if (want > 0xFFFFFF00ull) return sx_fail(ctx, SX_ERR_CAPACITY, "sx_process_window_dev: the window's insert pool would exceed 4 GiB; cut it into smaller windows");
        lo.cap_ins = (uint32_t)want;
    }
    if ((rc = take(ctx, SX_SLOT_WIN_LINK_TOTALS, 4, lo.totals))) return rc;
    lo.regions = b->regions;
    if ((rc = take(ctx, SX_SLOT_WIN_LINK_ALNS, (size_t)nA + 2, lo.alns))) return rc;
    if ((rc = take(ctx, SX_SLOT_WIN_LINK_SEGS, (size_t)lo.cap_segs + 32, lo.segs))) return rc;
    if ((rc = take(ctx, SX_SLOT_WIN_LINK_INS, (size_t)lo.cap_ins + SX_POOL_SLACK + 16, lo.ins))) return rc;
    if ((rc = take(ctx, SX_SLOT_WIN_K6_SEGS, (size_t)nS + 16, lo.k6_segs))) return rc;
    double* lnp(nullptr);
    if ((rc = take(ctx, SX_SLOT_WIN_LNP, (size_t)nA + 2, lnp))) return rc;
    uint32_t link_totals[2] = {0, 0};
    if (n)
    {
        if ((rc = sx_k8_run(ctx, &eb, &eo, nA, b->key_ins_off, b->key_ins, &lo, P.region, &launches))) return rc;
        SX_CUDA(ctx, cudaMemcpyAsync(link_totals, lo.totals, 8, cudaMemcpyDeviceToHost, st));
    }
    // ---------------------------------------------------------------------------------------------------------------- K1 scores
    SX_CUDA(ctx, mark(SX_WIN_ST_SCORE));
    if (n)
    {
        SX_CUDA(ctx, cudaStreamSynchronize(st));
        totals[3] = link_totals[0];
        totals[4] = link_totals[1];
        sx_align_batch ab;
        memset(&ab, 0, sizeof(ab));
        ab.n_regions = nr;
        ab.n_reads = n;
        ab.n_alns = nA;
        ab.n_segs = link_totals[0];
        ab.regions = b->regions;
        ab.read_len = b->read_len;
        ab.seq4 = b->seq4;
        ab.qual = b->qual;
        ab.ref = b->ref;
        ab.alns = lo.alns;
        ab.segs = lo.segs;
        ab.ins = lo.ins;
        ab.seq4_bytes = b->seq4_bytes;
        ab.qual_bytes = b->qual_bytes;
        ab.ref_bytes = b->ref_bytes;
        ab.ins_bytes = link_totals[1];
        ab.qual_bits = b->qual_bits == 4 ? 4u : 8u;
        memcpy(ab.qual_dict, b->qual_dict, 16);
        if ((rc = sx_k1_run(ctx, &ab, lnp, &launches))) return rc;
    }
    // ---------------------------------------------------------------------------------------------------------------- K6 score_indels
    SX_CUDA(ctx, mark(SX_WIN_ST_SCORE_INDELS));
    uint32_t n_rec_slots(0);
    if (n) SX_CUDA(ctx, cudaMemcpyAsync(&n_rec_slots, b->rec_off + n, 4, cudaMemcpyDeviceToHost, st));
    sx_score_indels_out so;
    memset(&so, 0, sizeof(so));
    if (n)
    {
        SX_CUDA(ctx, cudaStreamSynchronize(st));
        if ((rc = pick(ctx, S.recs, (size_t)n_rec_slots + 1, out->recs, so.recs))) return rc;
        if ((rc = pick(ctx, S.n_rec, (size_t)n + 1, out->n_rec, so.n_rec))) return rc;
        if ((rc = take(ctx, SX_SLOT_WIN_MAX_ALN, (size_t)n + 1, so.max_aln))) return rc;
        if ((rc = take(ctx, SX_SLOT_WIN_EVAL_ALN, (size_t)n + 1, so.eval_aln))) return rc;
        sx_score_indels_batch sb;
        memset(&sb, 0, sizeof(sb));
        sb.n_regions = nr;
        sb.n_reads = n;
        sb.n_alns = nA;
        sb.n_keys = b->n_keys;
        sb.region_read_off = b->region_read_off;
        sb.region_key_off = b->region_key_off;
        sb.keys = b->keys;
        sb.aln_off = eo.aln_off;
        sb.aln_pos = eo.aln_pos;
        sb.aln_seg_off = eo.aln_seg_off;
        sb.segs = lo.k6_segs;
        sb.aln_key_off = eo.aln_key_off;
        sb.aln_keys = eo.aln_keys;
        sb.read_len = b->read_len;
        sb.non_ambig = P.non_ambig;
        sb.read_flags = b->read_flags; // SX_SIF_FWD / SX_SIF_TIER1 are SX_PRF_FWD / SX_PRF_TIER1; the third SIF bit changes no output
        sb.rec_off = b->rec_off;
        sb.opts = b->score_opts;
        if ((rc = sx_k6_run(ctx, &sb, lnp, &so, &launches))) return rc;
    }
    // ---------------------------------------------------------------------------------------------------------------- K9 best alignments
    SX_CUDA(ctx, mark(SX_WIN_ST_CHOOSE));
    sx_realign_out ro;
    memset(&ro, 0, sizeof(ro));
    const uint32_t need_best(nS + 2u * n + n_raw_segs + 64u);
    ro.cap_segs = out->best_segs ? out->cap_best_segs : need_best;
    if ((rc = take(ctx, SX_SLOT_WIN_BEST_TOTALS, 4, ro.totals))) return rc;
    if ((rc = pick(ctx, SX_SLOT_WIN_BEST_SEG_OFF, (size_t)n + 2, out->best_seg_off, ro.seg_off))) return rc;
    if ((rc = pick(ctx, SX_SLOT_WIN_BEST_POS, (size_t)n + 1, out->best_pos, ro.pos))) return rc;
    if ((rc = pick(ctx, SX_SLOT_WIN_BEST_N_SEG, (size_t)n + 1, out->best_n_seg, ro.n_seg))) return rc;
    if ((rc = pick(ctx, SX_SLOT_WIN_REALIGN_STATUS, (size_t)n + 1, out->realign_status, ro.status))) return rc;
    if ((rc = take(ctx, SX_SLOT_WIN_BEST_ALN, (size_t)n + 1, ro.best_aln))) return rc;
    if ((rc = pick(ctx, SX_SLOT_WIN_BEST_SEGS, (size_t)ro.cap_segs + 16, out->best_segs, ro.segs))) return rc;
    if (n)
    {
        sx_realign_batch rb;
        memset(&rb, 0, sizeof(rb));
        rb.n_regions = nr;
        rb.n_reads = n;
        rb.n_alns = nA;
        rb.region_read_off = b->region_read_off;
        rb.region_key_off = b->region_key_off;
        rb.keys = b->keys;
        rb.aln_off = eo.aln_off;
        rb.aln_pos = eo.aln_pos;
        rb.aln_seg_off = eo.aln_seg_off;
        rb.segs = eo.segs;
        rb.aln_key_off = eo.aln_key_off;
        rb.aln_keys = eo.aln_keys;
        rb.read_len = b->read_len;
        rb.pin_flags = P.pin;
        rb.is_smoothed_alignments = b->score_opts.is_smoothed_alignments;
        rb.k4_kinds = 1;
        rb.smoothed_lnp_range = b->score_opts.smoothed_lnp_range;
        rb.raw_pos = b->raw_pos;
        rb.raw_seg_off = b->raw_seg_off;
        rb.raw_segs = b->raw_segs;
        if ((rc = sx_k9_run(ctx, &rb, lnp, &ro, P.region, &launches))) return rc;
    }
    // ---------------------------------------------------------------------------------------------------------------- K4 pile-up
    SX_CUDA(ctx, mark(SX_WIN_ST_PILEUP));
    sx_pileup_read* preads(nullptr);
    if ((rc = take(ctx, SX_SLOT_WIN_PILEUP_READS, (size_t)n + 2, preads))) return rc;
    sx_pileup_columns cols(out->cols);
    sx_pileup_reads_batch pb;
    memset(&pb, 0, sizeof(pb));
    uint64_t total_bases(0);
    int st_word(0);
    if (n)
    {
        sxp_pileup_reads_kernel<<<grid(n + 1), 128, 0, st>>>(*b, P, ro.pos, ro.seg_off, ro.segs, ro.status, preads);
        SX_CUDA(ctx, cudaGetLastError());
        ++launches;
        uint32_t best_total(0);
        SX_CUDA(ctx, cudaMemcpyAsync(maxima, P.maxima, 16, cudaMemcpyDeviceToHost, st));
        SX_CUDA(ctx, cudaMemcpyAsync(&best_total, ro.totals, 4, cudaMemcpyDeviceToHost, st));
        if ((rc = read_status(ctx, &st_word))) return rc;
        SX_CUDA(ctx, cudaStreamSynchronize(st));
        totals[5] = best_total;
        if (st_word & SX_ST_K9_CAP)
        {
            cudaMemsetAsync(ctx->d_status, 0, sizeof(int), st);
            if (totals_host) memcpy(totals_host, totals, sizeof(totals));
            return sx_fail(ctx, SX_ERR_CAPACITY, "sx_process_window_dev: cap_best_segs too small: %u segment slots needed", best_total);
        }
        if (st_word & SX_ST_K8_CAP)
        {
            cudaMemsetAsync(ctx->d_status, 0, sizeof(int), st);
            return sx_fail(ctx, SX_ERR_CAPACITY, "sx_process_window_dev: the linked alignments (%u segments, %u insert bytes) exceed their buffers", link_totals[0], link_totals[1]);
        }
    }
    {
        // the columns never hold more calls than the reads have bases
        total_bases = (uint64_t)b->seq4_bytes * 2u + 16u;
        const uint64_t cap_calls(cols.calls ? cols.calls_capacity : total_bases), cap_t2(cols.t2_calls ? cols.t2_capacity : (b->pileup_opts.useTier2Evidence || S.t2_all_bases ? total_bases : 64u));
        if ((rc = pick(ctx, S.site_off, (size_t)n_sites + 2, out->cols.site_off, cols.site_off))) return rc;
        if ((rc = pick(ctx, S.t2_off, (size_t)n_sites + 2, out->cols.t2_off, cols.t2_off))) return rc;
        if ((rc = pick(ctx, SX_SLOT_WIN_N_SPANDEL, (size_t)n_sites + 2, out->cols.n_spandel, cols.n_spandel))) return rc;
        if ((rc = pick(ctx, SX_SLOT_WIN_N_SUBMAPPED, (size_t)n_sites + 2, out->cols.n_submapped, cols.n_submapped))) return rc;
        if ((rc = pick(ctx, S.calls, (size_t)cap_calls + 16, out->cols.calls, cols.calls))) return rc;
        if ((rc = pick(ctx, S.t2_calls, (size_t)cap_t2 + 16, out->cols.t2_calls, cols.t2_calls))) return rc;
        cols.calls_capacity = cap_calls;
        cols.t2_capacity = cap_t2;
        pb.n_reads = n;
        pb.n_segs = totals[5];
        pb.reads = preads;
        pb.seq4 = b->seq4;
        pb.qual = b->qual;
        pb.segs = ro.segs;
        pb.ref = b->ref;
        pb.ref_begin = b->ref_begin;
        pb.ref_len = (uint32_t)std::min<uint64_t>(b->ref_bytes, 0xFFFFFFFFull);
        pb.report_begin = b->report_begin;
        pb.report_end = b->report_end;
        pb.cand_snv = b->cand_snv;
        pb.n_cand_snv = b->n_cand_snv;
        pb.max_ref_span = std::max<uint32_t>(1, maxima[2]);
        pb.max_read_len = b->max_read_len;
        pb.opts = b->pileup_opts;
        pb.buffer_pos = P.bpos;
        pb.max_pos_shift = maxima[1];
        pb.qual_bits = b->qual_bits == 4 ? 4u : 8u;
        memcpy(pb.qual_dict, b->qual_dict, 16);
        if ((rc = sx_k4_run(ctx, &pb, &cols, &launches)))
        {
            if (totals_host) memcpy(totals_host, totals, sizeof(totals));
            return rc;
        }
    }
    // ---------------------------------------------------------------------------------------------------------------- K2a site likelihoods
    SX_CUDA(ctx, mark(SX_WIN_ST_SITE_GL));
    if (b->do_site_gl && n_sites)
    {
        sx_digt_result* gl(nullptr);
        if ((rc = pick(ctx, SX_SLOT_WIN_SITE_GL, (size_t)n_sites + 1, out->site_gl, gl))) return rc;
        sx_pileup_batch k2;
        memset(&k2, 0, sizeof(k2));
        k2.n_sites = n_sites;
        k2.site_off = cols.site_off;
        k2.calls = cols.calls;
        k2.ref_base = b->ref + ((int64_t)b->report_begin - (int64_t)b->ref_begin);
        if ((int64_t)b->report_begin < (int64_t)b->ref_begin || (uint64_t)((int64_t)b->report_end - (int64_t)b->ref_begin) > b->ref_bytes)
            return sx_fail(ctx, SX_ERR_ARG, "sx_process_window_dev: the report range leaves the reference segment");
        if ((rc = sx_k2a_run(ctx, &k2, b->is_always_test, gl, &launches))) return rc;
        if (out->variant_sites)
        {
            const variant_site_sel sel = {gl, cols.site_off, b->report_begin};
            if ((rc = compact(ctx, sel, n_sites, SX_SLOT_WIN_VARIANT_CHUNKS, SX_SLOT_WIN_VARIANT_SUMS, out->variant_sites, out->cap_variant_sites, &totals[8], &launches)))
                return rc;
        }
    }
    else if (out->variant_sites)
        return sx_fail(ctx, SX_ERR_ARG, "sx_process_window_dev: variant_sites needs do_site_gl");
    SX_CUDA(ctx, mark(SX_WIN_N_STAGES));
    // ---------------------------------------------------------------------------------------------------------------- K4m metrics (the metrics entries)
    if (M.out)
    {
        if ((rc = sx_k4m_run(ctx, &pb, M.opts, M.out, &launches))) return rc;
        SX_CUDA(ctx, mark(SX_WIN_ST_METRICS + 1));
    }
    // ---------------------------------------------------------------------------------------------------------------- the end: one wait, the totals, the status
    uint32_t call_totals[2] = {0, 0};
    SX_CUDA(ctx, cudaMemcpyAsync(&call_totals[0], cols.site_off + n_sites, 4, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaMemcpyAsync(&call_totals[1], cols.t2_off + n_sites, 4, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaStreamSynchronize(st));
    totals[6] = call_totals[0];
    totals[7] = call_totals[1];
    if (out->totals) SX_CUDA(ctx, cudaMemcpyAsync(out->totals, totals, sizeof(totals), cudaMemcpyHostToDevice, st));
    if (totals_host) memcpy(totals_host, totals, sizeof(totals));
    float sum(0);
    for (int i = 0; i < SX_WIN_N_STAGES; ++i)
    {
        float ms(0);
        cudaEventElapsedTime(&ms, ctx->ev_win[i], ctx->ev_win[i + 1]);
        ctx->win_ms[i] = ms;
        sum += ms;
    }
    if (M.out)
    {
        float ms(0);
        cudaEventElapsedTime(&ms, ctx->ev_win[SX_WIN_ST_METRICS], ctx->ev_win[SX_WIN_ST_METRICS + 1]);
        ctx->win_ms[SX_WIN_ST_METRICS] = ms;
        sum += ms;
    }
    ctx->timing.kernel_ms = sum;
    ctx->timing.launches = launches;
    ctx->total_launches += launches;
    if (out->variant_sites && totals[8] > out->cap_variant_sites)
        return sx_fail(ctx, SX_ERR_CAPACITY, "sx_process_window_dev: %u variant sites, cap_variant_sites is %u", totals[8], out->cap_variant_sites);
    if (kept) *kept = win_kept{P.non_ambig, so.recs, so.n_rec, cols};
    return sx_check_status(ctx, "sx_process_window");
}
} // namespace

extern "C" int sx_process_window_dev(sx_ctx* ctx, const sx_window_batch* b, sx_window_out* out, uint32_t* totals_host)
{
    return window_pass(ctx, b, out, totals_host);
}

namespace
{
int check_window_metrics(sx_ctx* ctx, const char* what, const sx_pileup_metrics_opts* o)
{
    if (!o) return sx_fail(ctx, SX_ERR_ARG, "%s: NULL metrics options", what);
    if (o->mode != SX_PM_MAPQ && o->mode != SX_PM_GERMLINE && o->mode != SX_PM_SOMATIC)
        return sx_fail(ctx, SX_ERR_ARG, "%s: mode %u is not SX_PM_MAPQ, SX_PM_GERMLINE or SX_PM_SOMATIC", what, o->mode);
    if (o->full_len || o->full_off) return sx_fail(ctx, SX_ERR_ARG, "%s: full_len / full_off must be NULL (the window's reads are whole reads)", what);
    return SX_OK;
}
} // namespace

extern "C" int sx_process_window_metrics_dev(sx_ctx* ctx, const sx_window_batch* b, sx_window_out* out, uint32_t* totals_host, const sx_pileup_metrics_opts* mopts,
                                             sx_pileup_metrics_rec* metrics_dev)
{
    if (!ctx) return SX_ERR_ARG;
    if (!metrics_dev) return window_pass(ctx, b, out, totals_host);
    int rc;
    if ((rc = check_window_metrics(ctx, "sx_process_window_metrics_dev", mopts))) return rc;
    return window_pass(ctx, b, out, totals_host, WIN_SLOTS, nullptr, win_metrics{mopts, metrics_dev});
}

extern "C" int sx_last_window_metrics_timing(const sx_ctx* ctx, float* ms)
{
    if (!ctx || !ms) return SX_ERR_ARG;
    for (int i = 0; i <= SX_WIN_ST_METRICS; ++i) ms[i] = ctx->win_ms[i];
    return SX_OK;
}

// ---------------------------------------------------------------------------------------------------------------------------------------
// the somatic window pass: both samples through window_pass, then K2b, the SNV records, the link, K5b and the indel records
// ---------------------------------------------------------------------------------------------------------------------------------------
extern "C" int sx_last_somatic_window_timing(const sx_ctx* ctx, float* ms)
{
    if (!ctx || !ms) return SX_ERR_ARG;
    for (int i = 0; i < SX_SWIN_N_STAGES; ++i) ms[i] = ctx->swin_ms[i];
    return SX_OK;
}

namespace
{
// one sample's side of the link: the window batch's read arrays and the K6 records / 'N'-free counts its pass left
sx_indel_reads_sample indel_reads_sample_of(const sx_window_batch& b, const win_kept& k, const uint32_t* key_gid, const uint32_t* read_id)
{
    sx_indel_reads_sample s;
    memset(&s, 0, sizeof(s));
    s.n_regions = b.n_regions;
    s.n_reads = b.n_reads;
    s.n_keys = b.n_keys;
    s.region_read_off = b.region_read_off;
    s.region_key_off = b.region_key_off;
    s.key_gid = key_gid;
    s.rec_off = b.rec_off;
    s.recs = k.recs;
    s.n_rec = k.n_rec;
    s.read_len = b.read_len;
    s.non_ambig = k.non_ambig;
    s.read_flags = b.read_flags; // SX_SIF_TIER1 is SX_PRF_TIER1
    s.read_id = read_id;
    return s;
}

// a sample's tier1 (and with tier2 evidence its tier2) columns as K2b's batch
sx_pileup_batch somatic_pileup_of(const sx_pileup_columns& c, const uint32_t n_sites, const char* ref_base, const bool tier2)
{
    sx_pileup_batch p;
    memset(&p, 0, sizeof(p));
    p.n_sites = n_sites;
    p.site_off = c.site_off;
    p.calls = c.calls;
    p.t2_off = tier2 ? c.t2_off : nullptr;
    p.t2_calls = tier2 ? c.t2_calls : nullptr;
    p.ref_base = ref_base;
    return p;
}
} // namespace

namespace
{
// the somatic window pass; M[s].out non-NULL: K4m on sample s's pile-up batch at the end of its pass
int somatic_window_pass(sx_ctx* ctx, const sx_somatic_window_batch* sb, sx_somatic_window_out* so, uint32_t* totals_host, const char* what,
                        const win_metrics (&M)[2])
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    if (!sb || !so) return sx_fail(ctx, SX_ERR_ARG, "%s: NULL argument", what);
    const sx_window_batch &bn(sb->sample[0]), &bt(sb->sample[1]);
    for (int s = 0; s < 2; ++s)
    {
        const sx_window_batch& b(sb->sample[s]);
        if (b.do_site_gl) return sx_fail(ctx, SX_ERR_ARG, "%s: sample %d: do_site_gl must be 0 (strelka2 runs no germline site model)", what, s);
        if (so->sample[s].site_gl || so->sample[s].variant_sites) return sx_fail(ctx, SX_ERR_ARG, "%s: sample %d: site_gl / variant_sites must be NULL", what, s);
        if (b.n_keys && !sb->key_gid[s]) return sx_fail(ctx, SX_ERR_ARG, "%s: sample %d: NULL key_gid", what, s);
        if (b.report_end >= b.report_begin &&
            ((int64_t)b.report_begin < (int64_t)b.ref_begin || (uint64_t)((int64_t)b.report_end - (int64_t)b.ref_begin) > b.ref_bytes || !b.ref))
            return sx_fail(ctx, SX_ERR_ARG, "%s: sample %d: the report range leaves the reference segment", what, s);
    }
    if (bn.ref_begin != bt.ref_begin || bn.report_begin != bt.report_begin || bn.report_end != bt.report_end)
        return sx_fail(ctx, SX_ERR_ARG, "%s: the samples differ in ref_begin / report_begin / report_end", what);
    if (bn.pileup_opts.useTier2Evidence != bt.pileup_opts.useTier2Evidence || bn.pileup_opts.useTier2Evidence != sb->sindel_opts.useTier2Evidence)
        return sx_fail(ctx, SX_ERR_ARG, "%s: pileup_opts.useTier2Evidence of both samples must equal sindel_opts.useTier2Evidence", what);
    const sx_indel_loci& loci(sb->loci);
    int rc;
    if ((rc = sx_k6b_check_loci(ctx, what, &loci))) return rc;
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st(ctx->s_compute);
    const uint32_t n_sites(bn.report_end >= bn.report_begin ? (uint32_t)(bn.report_end - bn.report_begin) : 0u), n_loci(loci.n_loci);
    const bool tier2(sb->sindel_opts.useTier2Evidence != 0);
    sx_ssnv_result* site_snv(so->site_snv);
    sx_sindel_result* indel(so->indel);
    if (!site_snv && (rc = take(ctx, SX_SLOT_SWIN_SITE_SNV, (size_t)n_sites + 1, site_snv))) return rc;
    if (!indel && (rc = take(ctx, SX_SLOT_SWIN_INDEL, (size_t)n_loci + 1, indel))) return rc;
    sx_indel_reads_out lo;
    if ((rc = sx_k6b_own_out(ctx, n_loci, &lo))) return rc;
    {
        const sx_sindel_batch kb(sx_sindel_batch_of(&loci, &lo));
        if ((rc = sx_k5b_check(ctx, what, &sb->sindel_opts, &kb, sb->err_prob, sb->n_err, indel))) return rc;
    }
    for (int i = 0; i <= SX_SWIN_N_STAGES; ++i)
        if (!ctx->ev_swin[i]) SX_CUDA(ctx, cudaEventCreate(&ctx->ev_swin[i]));
    auto mark = [&](int i) { return cudaEventRecord(ctx->ev_swin[i], st); };
    unsigned launches(0), pass_launches(0); // (the passes add theirs to ctx->total_launches themselves)
    float metrics_ms(0);                    // (the metrics stages, inside the samples' passes)
    uint32_t totals[SX_SWIN_TOTALS] = {0, 0, 0, 0};

    // ---------------------------------------------------------------------------------------------------------------- the two chains
    // The normal sample's results that the stages below read go to the SX_SLOT_SWIN_* bank, so the tumor sample's pass leaves them be.
    win_kept kept[2];
    // A sample's SX_ERR_CAPACITY (an output array of out.sample[s] too small) leaves that pass's totals in out.sample[s].totals, as
    // sx_process_window_dev's totals_host would.
    const auto sample_pass = [&](const int s, const win_slots& slots) -> int {
        uint32_t wt[SX_WIN_TOTALS] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
        const int r(window_pass(ctx, &sb->sample[s], &so->sample[s], wt, slots, &kept[s], M[s]));
        if (M[s].out) metrics_ms += ctx->win_ms[SX_WIN_ST_METRICS];
        if (r == SX_ERR_CAPACITY && so->sample[s].totals) cudaMemcpy(so->sample[s].totals, wt, sizeof(wt), cudaMemcpyHostToDevice);
        pass_launches += ctx->timing.launches;
        return r;
    };
    SX_CUDA(ctx, mark(SX_SWIN_ST_NORMAL));
    if ((rc = sample_pass(0, SWIN_NORMAL_SLOTS))) return rc;
    SX_CUDA(ctx, mark(SX_SWIN_ST_TUMOR));
    if ((rc = sample_pass(1, SWIN_TUMOR_SLOTS))) return rc;
    // ---------------------------------------------------------------------------------------------------------------- K2b and the SNV records
    SX_CUDA(ctx, mark(SX_SWIN_ST_SITE_SNV));
    const char* ref_base(bn.ref + ((int64_t)bn.report_begin - (int64_t)bn.ref_begin));
    const sx_pileup_batch pn(somatic_pileup_of(kept[0].cols, n_sites, ref_base, tier2)), pt(somatic_pileup_of(kept[1].cols, n_sites, ref_base, tier2));
    if (n_sites && (rc = sx_k2b_run(ctx, &pn, &pt, sb->snv_forced_output, site_snv, sb->is_compute_nonsomatic != 0, &launches))) return rc;
    SX_CUDA(ctx, mark(SX_SWIN_ST_SNV_CALLS));
    if (n_sites && so->snv_calls)
    {
        const somatic_site_sel sel = {site_snv, sb->snv_forced_output, ref_base, pn.site_off, pt.site_off, bn.report_begin};
        if ((rc = compact(ctx, sel, n_sites, SX_SLOT_SWIN_SNV_CHUNKS, SX_SLOT_SWIN_SNV_SUMS, so->snv_calls, so->cap_snv_calls, &totals[0], &launches))) return rc;
    }
    // ---------------------------------------------------------------------------------------------------------------- link, K5b, the indel records
    SX_CUDA(ctx, mark(SX_SWIN_ST_LINK));
    if (n_loci)
    {
        const sx_indel_reads_sample rn(indel_reads_sample_of(bn, kept[0], sb->key_gid[0], sb->read_id[0])), rt(indel_reads_sample_of(bt, kept[1], sb->key_gid[1], sb->read_id[1]));
        if ((rc = sx_k6b_run(ctx, what, &rn, &rt, &loci, &lo, &totals[2], true, &launches))) return rc;
        SX_CUDA(ctx, mark(SX_SWIN_ST_INDEL));
        if ((rc = sx_sindel_from_links_run(ctx, &sb->sindel_opts, &loci, &lo, sb->err_prob, sb->n_err, indel, &launches))) return rc;
    }
    else SX_CUDA(ctx, mark(SX_SWIN_ST_INDEL));
    SX_CUDA(ctx, mark(SX_SWIN_ST_INDEL_CALLS));
    if (n_loci && so->indel_calls)
    {
        const somatic_indel_sel sel = {indel, loci.is_forced_output, lo.status, lo.read_off};
        if ((rc = compact(ctx, sel, n_loci, SX_SLOT_SWIN_INDEL_CHUNKS, SX_SLOT_SWIN_INDEL_SUMS, so->indel_calls, so->cap_indel_calls, &totals[1], &launches))) return rc;
    }
    SX_CUDA(ctx, mark(SX_SWIN_N_STAGES));
    // ---------------------------------------------------------------------------------------------------------------- the end: one wait, the totals, the status
    SX_CUDA(ctx, cudaStreamSynchronize(st));
    if (so->totals) SX_CUDA(ctx, cudaMemcpyAsync(so->totals, totals, sizeof(totals), cudaMemcpyHostToDevice, st));
    if (totals_host) memcpy(totals_host, totals, sizeof(totals));
    float sum(0);
    for (int i = 0; i < SX_SWIN_N_STAGES; ++i)
    {
        float ms(0);
        cudaEventElapsedTime(&ms, ctx->ev_swin[i], ctx->ev_swin[i + 1]);
        ctx->swin_ms[i] = ms;
        sum += ms;
    }
    ctx->swin_ms[SX_SWIN_ST_METRICS] = metrics_ms;
    ctx->timing.kernel_ms = sum;
    ctx->timing.launches = pass_launches + launches;
    ctx->total_launches += launches;
    if ((rc = sx_check_status(ctx, what, SX_ST_K6B_ID))) return rc;
    if (so->snv_calls && totals[0] > so->cap_snv_calls)
        return sx_fail(ctx, SX_ERR_CAPACITY, "%s: %u somatic SNV records, cap_snv_calls is %u", what, totals[0], so->cap_snv_calls);
    if (so->indel_calls && totals[1] > so->cap_indel_calls)
        return sx_fail(ctx, SX_ERR_CAPACITY, "%s: %u somatic indel records, cap_indel_calls is %u", what, totals[1], so->cap_indel_calls);
    return SX_OK;
}

} // namespace

extern "C" int sx_process_somatic_window_dev(sx_ctx* ctx, const sx_somatic_window_batch* sb, sx_somatic_window_out* so, uint32_t* totals_host)
{
    const win_metrics none[2] = {{nullptr, nullptr}, {nullptr, nullptr}};
    return somatic_window_pass(ctx, sb, so, totals_host, "sx_process_somatic_window_dev", none);
}

extern "C" int sx_process_somatic_window_metrics_dev(sx_ctx* ctx, const sx_somatic_window_batch* sb, sx_somatic_window_out* so, uint32_t* totals_host,
                                                     const sx_pileup_metrics_opts* const mopts[2], sx_pileup_metrics_rec* const metrics_dev[2])
{
    if (!ctx) return SX_ERR_ARG;
    const char* what("sx_process_somatic_window_metrics_dev");
    win_metrics M[2] = {{nullptr, nullptr}, {nullptr, nullptr}};
    for (int s = 0; s < 2 && metrics_dev; ++s)
    {
        if (!metrics_dev[s]) continue;
        int rc;
        if ((rc = check_window_metrics(ctx, what, mopts ? mopts[s] : nullptr))) return rc;
        M[s] = win_metrics{mopts[s], metrics_dev[s]};
    }
    ctx->swin_ms[SX_SWIN_ST_METRICS] = 0;
    return somatic_window_pass(ctx, sb, so, totals_host, what, M);
}

extern "C" int sx_last_somatic_window_metrics_timing(const sx_ctx* ctx, float* ms)
{
    if (!ctx || !ms) return SX_ERR_ARG;
    for (int i = 0; i <= SX_SWIN_ST_METRICS; ++i) ms[i] = ctx->swin_ms[i];
    return SX_OK;
}

// ---------------------------------------------------------------------------------------------------------------------------------------
// host arrays in, host arrays out
// ---------------------------------------------------------------------------------------------------------------------------------------
extern "C" int sx_process_window(sx_ctx* ctx, const sx_window_batch* b, sx_window_out* out, uint32_t* totals_host)
{
    if (!ctx) return SX_ERR_ARG;
    if (!b || !out) return sx_fail(ctx, SX_ERR_ARG, "sx_process_window: NULL argument");
    if (b->n_reads && (!b->region_read_off || !b->region_key_off || !b->raw_seg_off || !b->use_key_off || !b->rec_off || !b->regions || (b->n_keys && !b->key_ins_off)))
        return sx_fail(ctx, SX_ERR_ARG, "sx_process_window: NULL array");
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st(ctx->s_compute);
    const uint32_t n(b->n_reads), nr(b->n_regions), nk(b->n_keys);
    const uint32_t n_sites((uint32_t)(b->report_end - b->report_begin));
    sx_window_batch d(*b);
    int rc;
    float h2d_ms(0), d2h_ms(0);
    cudaEvent_t e0(ctx->ev_a), e1(ctx->ev_b);
    SX_CUDA(ctx, cudaEventRecord(e0, st));
    const size_t n_raw(n ? b->raw_seg_off[n] : 0), n_use(n ? b->use_key_off[n] : 0), ins_bytes(nk ? b->key_ins_off[nk] : 0);
    // An array the caller left NULL (key_ins_off without keys, every array of an empty window) is not copied; its buffer is still passed on.
    const auto up = [&](sx_slot slot, const auto* src, size_t count, auto& dst) -> int {
        return src ? sx_upload(ctx, slot, src, count, dst, 80) : sx_take(ctx, slot, count, dst, 80);
    };
    if ((rc = up(SX_SLOT_WUP_REGION_READ_OFF, b->region_read_off, (size_t)nr + 1, d.region_read_off))) return rc;
    if ((rc = up(SX_SLOT_WUP_REGION_KEY_OFF, b->region_key_off, (size_t)nr + 1, d.region_key_off))) return rc;
    if ((rc = up(SX_SLOT_WUP_KEYS, b->keys, nk, d.keys))) return rc;
    if (b->key_hap && (rc = up(SX_SLOT_WUP_KEY_HAP, b->key_hap, nk, d.key_hap))) return rc;
    if ((rc = up(SX_SLOT_WUP_KEY_INS_OFF, b->key_ins_off, (size_t)nk + 1, d.key_ins_off))) return rc;
    if ((rc = up(SX_SLOT_WUP_KEY_INS, b->key_ins, ins_bytes, d.key_ins))) return rc;
    if ((rc = up(SX_SLOT_WUP_REALIGN_BEGIN, b->realign_begin, nr, d.realign_begin))) return rc;
    if ((rc = up(SX_SLOT_WUP_REALIGN_END, b->realign_end, nr, d.realign_end))) return rc;
    if ((rc = up(SX_SLOT_WUP_RAW_POS, b->raw_pos, n, d.raw_pos))) return rc;
    if ((rc = up(SX_SLOT_WUP_RAW_SEG_OFF, b->raw_seg_off, (size_t)n + 1, d.raw_seg_off))) return rc;
    if ((rc = up(SX_SLOT_WUP_RAW_SEGS, b->raw_segs, n_raw, d.raw_segs))) return rc;
    if ((rc = up(SX_SLOT_WUP_READ_LEN, b->read_len, n, d.read_len))) return rc;
    if ((rc = up(SX_SLOT_WUP_READ_FLAGS, b->read_flags, n, d.read_flags))) return rc;
    if ((rc = up(SX_SLOT_WUP_MAPQ, b->mapq, n, d.mapq))) return rc;
    if ((rc = up(SX_SLOT_WUP_USE_KEY_OFF, b->use_key_off, (size_t)n + 1, d.use_key_off))) return rc;
    if ((rc = up(SX_SLOT_WUP_USE_KEYS, b->use_keys, n_use, d.use_keys))) return rc;
    if ((rc = up(SX_SLOT_WUP_REC_OFF, b->rec_off, (size_t)n + 1, d.rec_off))) return rc;
    if ((rc = up(SX_SLOT_WUP_REGIONS, b->regions, (size_t)nr + 1, d.regions))) return rc;
    if ((rc = up(SX_SLOT_WUP_SEQ4, b->seq4, b->seq4_bytes, d.seq4))) return rc;
    if ((rc = up(SX_SLOT_WUP_QUAL, b->qual, b->qual_bytes, d.qual))) return rc;
    if ((rc = up(SX_SLOT_WUP_REF, b->ref, b->ref_bytes, d.ref))) return rc;
    if (b->cand_snv && (rc = up(SX_SLOT_WUP_CAND_SNV, b->cand_snv, b->n_cand_snv, d.cand_snv))) return rc;
    SX_CUDA(ctx, cudaEventRecord(e1, st));
    // device outputs for whatever the caller wants back
    sx_window_out o;
    memset(&o, 0, sizeof(o));
    const size_t n_slots(n ? b->rec_off[n] : 0);
    const auto want = [&](const void* host, sx_slot slot, size_t count, auto*& dev) -> int { return host ? sx_take(ctx, slot, count, dev, 80) : SX_OK; };
    if ((rc = want(out->gate, SX_SLOT_WDN_GATE, n, o.gate))) return rc;
    if ((rc = want(out->enum_status, SX_SLOT_WDN_ENUM_STATUS, n, o.enum_status))) return rc;
    if ((rc = want(out->realign_status, SX_SLOT_WDN_REALIGN_STATUS, n, o.realign_status))) return rc;
    if ((rc = want(out->best_pos, SX_SLOT_WDN_BEST_POS, n, o.best_pos))) return rc;
    if ((rc = want(out->best_seg_off, SX_SLOT_WDN_BEST_SEG_OFF, (size_t)n + 1, o.best_seg_off))) return rc;
    if ((rc = want(out->best_n_seg, SX_SLOT_WDN_BEST_N_SEG, n, o.best_n_seg))) return rc;
    if ((rc = want(out->best_segs, SX_SLOT_WDN_BEST_SEGS, out->cap_best_segs, o.best_segs))) return rc;
    o.cap_best_segs = out->cap_best_segs;
    if ((rc = want(out->recs, SX_SLOT_WDN_RECS, n_slots + 1, o.recs))) return rc;
    if ((rc = want(out->n_rec, SX_SLOT_WDN_N_REC, n, o.n_rec))) return rc;
    if ((rc = want(out->cols.site_off, SX_SLOT_WDN_SITE_OFF, (size_t)n_sites + 1, o.cols.site_off))) return rc;
    if ((rc = want(out->cols.t2_off, SX_SLOT_WDN_T2_OFF, (size_t)n_sites + 1, o.cols.t2_off))) return rc;
    if ((rc = want(out->cols.n_spandel, SX_SLOT_WDN_N_SPANDEL, n_sites, o.cols.n_spandel))) return rc;
    if ((rc = want(out->cols.n_submapped, SX_SLOT_WDN_N_SUBMAPPED, n_sites, o.cols.n_submapped))) return rc;
    if ((rc = want(out->cols.calls, SX_SLOT_WDN_CALLS, out->cols.calls_capacity, o.cols.calls))) return rc;
    if ((rc = want(out->cols.t2_calls, SX_SLOT_WDN_T2_CALLS, out->cols.t2_capacity, o.cols.t2_calls))) return rc;
    o.cols.calls_capacity = out->cols.calls_capacity;
    o.cols.t2_capacity = out->cols.t2_capacity;
    if ((rc = want(out->site_gl, SX_SLOT_WDN_SITE_GL, n_sites, o.site_gl))) return rc;
    if ((rc = want(out->variant_sites, SX_SLOT_WDN_VARIANT_SITES, out->cap_variant_sites, o.variant_sites))) return rc;
    o.cap_variant_sites = out->cap_variant_sites;
    uint32_t totals[SX_WIN_TOTALS];
    memset(totals, 0, sizeof(totals));
    rc = window_pass(ctx, &d, &o, totals);
    if (totals_host) memcpy(totals_host, totals, sizeof(totals));
    if (rc) return rc;
    const float kernel_ms(ctx->timing.kernel_ms);
    const uint32_t launches(ctx->timing.launches);
    cudaEventElapsedTime(&h2d_ms, e0, e1);
    SX_CUDA(ctx, cudaEventRecord(e0, st));
    const auto down = [&](auto* host, const auto* dev, size_t count) -> int { return host ? sx_download(ctx, host, dev, count) : SX_OK; }; // (what the caller asked for)
    if ((rc = down(out->gate, o.gate, n))) return rc;
    if ((rc = down(out->enum_status, o.enum_status, n))) return rc;
    if ((rc = down(out->realign_status, o.realign_status, n))) return rc;
    if ((rc = down(out->best_pos, o.best_pos, n))) return rc;
    if ((rc = down(out->best_seg_off, o.best_seg_off, (size_t)n + 1))) return rc;
    if ((rc = down(out->best_n_seg, o.best_n_seg, n))) return rc;
    if ((rc = down(out->best_segs, o.best_segs, totals[5]))) return rc;
    if ((rc = down(out->recs, o.recs, n_slots))) return rc;
    if ((rc = down(out->n_rec, o.n_rec, n))) return rc;
    if ((rc = down(out->cols.site_off, o.cols.site_off, (size_t)n_sites + 1))) return rc;
    if ((rc = down(out->cols.t2_off, o.cols.t2_off, (size_t)n_sites + 1))) return rc;
    if ((rc = down(out->cols.n_spandel, o.cols.n_spandel, n_sites))) return rc;
    if ((rc = down(out->cols.n_submapped, o.cols.n_submapped, n_sites))) return rc;
    if ((rc = down(out->cols.calls, o.cols.calls, totals[6]))) return rc;
    if ((rc = down(out->cols.t2_calls, o.cols.t2_calls, totals[7]))) return rc;
    if ((rc = down(out->site_gl, o.site_gl, n_sites))) return rc;
    if ((rc = down(out->variant_sites, o.variant_sites, std::min(totals[8], out->cap_variant_sites)))) return rc;
    if (out->totals) memcpy(out->totals, totals, sizeof(totals));
    SX_CUDA(ctx, cudaEventRecord(e1, st));
    SX_CUDA(ctx, cudaStreamSynchronize(st));
    cudaEventElapsedTime(&d2h_ms, e0, e1);
    ctx->timing.kernel_ms = kernel_ms;
    ctx->timing.h2d_ms = h2d_ms;
    ctx->timing.d2h_ms = d2h_ms;
    ctx->timing.launches = launches;
    return SX_OK;
}
