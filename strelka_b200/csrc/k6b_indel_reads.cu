// k6b_indel_reads.cu -- K6b indel_reads: K6's per-read records regrouped into K5b's per-locus read lists, in device memory.
//
// Replaces (include/strelka_b200.h, "K6b indel_reads") the transpose the reference's containers do implicitly:
//   starling_common/starling_read_align_score_indels.cpp:1071   read_path_lnp[readId] = ReadPathScores(...)
//   starling_common/IndelData.hh:262                             the std::map the somatic caller walks
//   applications/strelka/strelka_pos_processor.cpp:305-348       process_pos_indel_somatic, its reader
//
// Shape of the work: every 32-byte record is read, one in a few becomes a 24-byte entry somewhere else -- no arithmetic, so the floor is
// the bytes (tools/indel_reads_leg.py counts them).  A CSR producer like K7b and K9: count -> scan (sx_scan) -> write, with a sort between.
//   k6b_locus_table_kernel  id -> locus as a dense table of n_gid words.  A binary search of loci.gid would cost ~20 dependent loads per
//                           record, twice (count and scatter), against one load here; the table is an eighth of the gid_key array the
//                           caller already holds, so an id space too sparse for it is too sparse for the ABI.
//   the list builder        (k6_lists.cuh) count, scan, scatter and sort into segments 2 * locus + sample, one warp per locus in the sort;
//                           its hook (k6b_hook) gathers the alternates' ids into an ascending set of at most 16 and writes each locus's status
//   scan                    of the unflagged loci's counts, in place in read_off and alt_off, -> totals; one 8-byte round trip checks
//                           the capacities
//   k6b_write_kernel        one warp per locus: the table rows from gid_key, and every entry (k6b_entry) at its sorted place
// The body is k6b_core.cuh.
#include "k6_lists.cuh"

namespace
{
constexpr int K6B_THREADS = 128;
constexpr int K6B_WARPS = K6B_THREADS / 32;
constexpr unsigned FULL = 0xffffffffu;
static_assert(SX_ST_INDEL_READS_DUP == SX_INDEL_READS_ST_DUP_READ, "the per-locus duplicate status of K6b is its status bit");

__global__ void k6b_locus_table_kernel(const sx_indel_loci loci, uint32_t* __restrict__ locus_of, int* __restrict__ status)
{
    for (uint32_t l = blockIdx.x * blockDim.x + threadIdx.x; l < loci.n_loci; l += gridDim.x * blockDim.x)
    {
        const uint32_t id(loci.gid[l]);
        if (id < loci.n_gid && (l == 0 || loci.gid[l - 1] < id)) locus_of[id] = l; // strictly ascending: no two loci store to one word
        else atomicOr(status, SX_ST_K6B_ID);
    }
}

// K6b's part of the list builder's sort: each locus's ascending alternate ids (alt_ids[16 * locus ..]), its status, and the counts the second
// scan runs over (read_off[2 * locus + sample], alt_off[locus]; 0 for a flagged locus)
struct k6b_hook
{
    static constexpr uint32_t n_samples = 2;
    struct warp_smem
    {
        uint32_t set[SX_SINDEL_MAX_ALTS], n, over;
    };
    k6b_view v;
    uint32_t* alt_ids;
    sx_indel_reads_out o;

    __device__ void begin(warp_smem& w, const uint32_t lane) const
    {
        if (lane == 0) w.n = w.over = 0;
        __syncwarp();
    }
    // the ids this segment's entries name as alternates, into the locus's set (lane 0 inserts, one new id per round)
    __device__ uint32_t segment(warp_smem& w, uint32_t, const uint32_t sample, const uint32_t base, const uint32_t n, const k6l_pairs& P, const uint32_t lane) const
    {
        const sx_indel_reads_sample& s(v.s[sample]);
        uint32_t bad(0);
        for (uint32_t i0 = 0; i0 < n && !w.over; i0 += 32)
        {
            uint32_t ids[2] = {K6B_NONE, K6B_NONE};
            if (i0 + lane < n)
            {
                const sx_read_indel_score& rec(s.recs[P.rec[base + i0 + lane]]);
                if (rec.n_alt) k6b_alt_ids(s, v.loci.n_gid, k6b_region_of(s, P.read[base + i0 + lane]), rec, ids, bad);
            }
            for (uint32_t a = 0; a < 2; ++a)
                for (;;)
                {
                    bool need(ids[a] != K6B_NONE && !w.over);
                    for (uint32_t k = 0; need && k < w.n; ++k) need = w.set[k] != ids[a];
                    const unsigned m(__ballot_sync(FULL, need));
                    if (!m) break;
                    const uint32_t id(__shfl_sync(FULL, ids[a], __ffs(m) - 1));
                    if (lane == 0 && !k6b_set_insert(w.set, w.n, id)) w.over = 1;
                    __syncwarp();
                }
        }
        return bad;
    }
    __device__ void end(warp_smem& w, const uint32_t l, const bool dup, const uint32_t* pair_off, const uint32_t lane) const
    {
        const uint32_t st((dup ? SX_INDEL_READS_ST_DUP_READ : 0u) | (w.over ? SX_SINDEL_ST_CAP : 0u));
        const uint32_t n_alts(st ? 0u : w.n);
        if (lane < n_alts) alt_ids[(size_t)SX_SINDEL_MAX_ALTS * l + lane] = w.set[lane];
        if (lane < 2) o.read_off[2 * l + lane] = st ? 0u : pair_off[2 * l + lane + 1] - pair_off[2 * l + lane];
        if (lane == 0)
        {
            o.status[l] = st;
            o.alt_off[l] = n_alts;
        }
        __syncwarp();
    }
};

__global__ void __launch_bounds__(K6B_THREADS) k6b_write_kernel(const k6b_view v, const uint32_t* __restrict__ pair_off, const k6l_pairs P, const uint32_t* __restrict__ alt_ids,
                                                               const sx_indel_reads_out o)
{
    const uint32_t lane(threadIdx.x & 31), warp(threadIdx.x >> 5);
    for (uint32_t l = blockIdx.x * K6B_WARPS + warp; l < v.loci.n_loci; l += gridDim.x * K6B_WARPS)
    {
        if (o.status[l]) continue;
        const uint32_t a0(o.alt_off[l]), n_alts(o.alt_off[l + 1] - a0);
        const uint32_t* ids(alt_ids + (size_t)SX_SINDEL_MAX_ALTS * l);
        if (lane < n_alts) o.alts[a0 + lane] = v.loci.gid_key[ids[lane]];
        for (uint32_t sample = 0; sample < 2; ++sample)
        {
            const sx_indel_reads_sample& s(v.s[sample]);
            const uint32_t base(pair_off[2 * l + sample]), n(pair_off[2 * l + sample + 1] - base), out0(o.read_off[2 * l + sample]);
            for (uint32_t i = lane; i < n; i += 32)
            {
                const uint32_t j(base + P.order[base + i]);
                o.reads[out0 + i] = k6b_entry(s, v.loci.n_gid, P.read[j], s.recs[P.rec[j]], ids, n_alts);
            }
        }
    }
}

// a flagged locus's result: its status and nothing else
__global__ void k6b_flag_results_kernel(const uint32_t n_loci, const uint32_t* __restrict__ loc_status, sx_sindel_result* __restrict__ out)
{
    for (uint32_t l = blockIdx.x * blockDim.x + threadIdx.x; l < n_loci; l += gridDim.x * blockDim.x)
    {
        const uint32_t st(loc_status[l]);
        if (!st) continue;
        uint32_t* w(reinterpret_cast<uint32_t*>(out + l));
        for (uint32_t i = 0; i < sizeof(sx_sindel_result) / 4; ++i) w[i] = 0u;
        out[l].status = st;
    }
}

int k6b_check(sx_ctx* ctx, const char* what, const sx_indel_reads_sample* normal, const sx_indel_reads_sample* tumor, const sx_indel_loci* loci)
{
    int rc;
    if ((rc = sx_k6b_check_sample(ctx, what, normal)) || (rc = sx_k6b_check_sample(ctx, what, tumor))) return rc;
    return sx_k6b_check_loci(ctx, what, loci);
}

int k6b_check_out(sx_ctx* ctx, const char* what, const sx_indel_reads_out* o)
{
    if (!o || !o->alt_off || !o->read_off || !o->totals) return sx_fail(ctx, SX_ERR_ARG, "%s: NULL output array", what);
    return SX_OK;
}

} // namespace

int sx_k6b_check_sample(sx_ctx* ctx, const char* what, const sx_indel_reads_sample* s)
{
    if (!s) return sx_fail(ctx, SX_ERR_ARG, "%s: NULL argument", what);
    if (s->n_reads == 0) return SX_OK;
    if (!s->region_read_off || !s->region_key_off || !s->rec_off || !s->recs || !s->n_rec || !s->read_len || !s->non_ambig || !s->read_flags || (s->n_keys && !s->key_gid))
        return sx_fail(ctx, SX_ERR_ARG, "%s: NULL sample array", what);
    if (s->n_regions == 0) return sx_fail(ctx, SX_ERR_ARG, "%s: reads without a region", what);
    return SX_OK;
}

int sx_k6b_check_loci(sx_ctx* ctx, const char* what, const sx_indel_loci* loci)
{
    if (!loci) return sx_fail(ctx, SX_ERR_ARG, "%s: NULL argument", what);
    if (loci->n_loci && (!loci->gid || !loci->key || !loci->is_forced_output || !loci->err_idx || !loci->gid_key || loci->n_gid == 0))
        return sx_fail(ctx, SX_ERR_ARG, "%s: NULL loci array", what);
    if (loci->n_loci > 0x7fffffffu) return sx_fail(ctx, SX_ERR_RANGE, "%s: more than 2^31 - 1 loci", what);
    return SX_OK;
}

// The stage's launcher, beside its kernels like sx_k6_run: everything is enqueued on the compute stream, with two small round trips (the
// list builder's, then the output totals).  own_out: the entry and table arrays are taken from the context's SX_SLOT_K6B_OUT_* buffers once
// the totals are known, instead of checked against the caller's capacities.
int sx_k6b_run(sx_ctx* ctx, const char* what, const sx_indel_reads_sample* normal, const sx_indel_reads_sample* tumor, const sx_indel_loci* loci, sx_indel_reads_out* o,
            uint32_t* totals_host, const bool own_out, unsigned* launches)
{
    cudaStream_t st(ctx->s_compute);
    const uint32_t n_loci(loci->n_loci), n2(2 * n_loci);
    uint32_t h_totals[2] = {0, 0};
    int rc;
    if (n_loci == 0)
    {
        SX_CUDA(ctx, cudaMemsetAsync(o->totals, 0, 8, st));
        SX_CUDA(ctx, cudaMemsetAsync(o->read_off, 0, 4, st));
        SX_CUDA(ctx, cudaMemsetAsync(o->alt_off, 0, 4, st));
        if (totals_host) totals_host[0] = totals_host[1] = 0;
        return SX_OK;
    }
    if (!o->status) return sx_fail(ctx, SX_ERR_ARG, "%s: NULL output array", what);
    uint32_t *locus_of(nullptr), *alt_ids(nullptr);
    if ((rc = sx_take(ctx, SX_SLOT_K6B_LOCUS_OF, loci->n_gid, locus_of, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K6B_ALT_IDS, (size_t)SX_SINDEL_MAX_ALTS * n_loci, alt_ids, 16))) return rc;

    k6b_view v;
    v.s[0] = *normal;
    v.s[1] = *tumor;
    v.loci = *loci;
    v.locus_of = locus_of;
    SX_CUDA(ctx, cudaMemsetAsync(locus_of, 0xFF, (size_t)loci->n_gid * 4, st));
    k6b_locus_table_kernel<<<k6l_grid(ctx, n_loci, 256), 256, 0, st>>>(*loci, locus_of, ctx->d_status);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 1;
    k6l_lists L;
    if ((rc = k6l_build(ctx, what, v, n_loci, k6b_hook{v, alt_ids, *o}, &L, launches))) return rc;
    const sx_scan_set out = {2, {{o->read_off, n2, SX_SCAN_EXCLUSIVE | SX_SCAN_CLOSE, o->totals}, {o->alt_off, n_loci, SX_SCAN_EXCLUSIVE | SX_SCAN_CLOSE, o->totals + 1}}};
    if ((rc = sx_scan(ctx, SX_SLOT_K6L_SUMS, out, launches))) return rc;
    SX_CUDA(ctx, cudaMemcpyAsync(h_totals, o->totals, 8, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaStreamSynchronize(st));
    if (totals_host)
    {
        totals_host[0] = h_totals[0];
        totals_host[1] = h_totals[1];
    }
    if (own_out)
    {
        if ((rc = sx_take(ctx, SX_SLOT_K6B_OUT_READS, h_totals[0], o->reads, 16))) return rc;
        if ((rc = sx_take(ctx, SX_SLOT_K6B_OUT_ALTS, h_totals[1], o->alts, 16))) return rc;
        o->cap_reads = h_totals[0];
        o->cap_alts = h_totals[1];
    }
    if (h_totals[0] > o->cap_reads || h_totals[1] > o->cap_alts)
        return sx_fail(ctx, SX_ERR_CAPACITY, "%s: output capacity too small: %u entries, %u alternates needed", what, h_totals[0], h_totals[1]);
    if ((h_totals[0] && !o->reads) || (h_totals[1] && !o->alts)) return sx_fail(ctx, SX_ERR_ARG, "%s: NULL output array", what);
    k6b_write_kernel<<<k6l_grid(ctx, n_loci, K6B_WARPS), K6B_THREADS, 0, st>>>(v, L.off, L.P, alt_ids, *o);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 1;
    return SX_OK;
}

namespace
{
template <typename T> bool k6b_ends_at(const T* off, const uint32_t n, const uint32_t end) { return n == 0 || (off[0] == 0 && off[n] == end); }
} // namespace

// host staging of one sample: slots base .. base + 9
int sx_k6b_upload_sample(sx_ctx* ctx, const char* what, const sx_indel_reads_sample* h, const int base, const uint32_t n_gid, sx_indel_reads_sample* d)
{
    *d = *h;
    if (h->n_reads == 0) return SX_OK;
    const size_t n(h->n_reads), n_slots(h->rec_off[n]);
    if (!k6b_ends_at(h->region_read_off, h->n_regions, h->n_reads) || !k6b_ends_at(h->region_key_off, h->n_regions, h->n_keys))
        return sx_fail(ctx, SX_ERR_ARG, "%s: offset arrays do not end at n_reads / n_keys", what);
    for (size_t r = 0; r < n; ++r)
        if (h->rec_off[r] > h->rec_off[r + 1] || h->n_rec[r] > h->rec_off[r + 1] - h->rec_off[r]) return sx_fail(ctx, SX_ERR_ARG, "%s: read %zu: n_rec past its record slots", what, r);
    for (uint32_t k = 0; k < h->n_keys; ++k)
        if (h->key_gid[k] >= n_gid) return sx_fail(ctx, SX_ERR_ARG, "%s: window entry %u: id %u past n_gid (%u)", what, k, h->key_gid[k], n_gid);
    int rc;
    if ((rc = sx_upload(ctx, sx_host_slot(base + 0), h->region_read_off, (size_t)h->n_regions + 1, d->region_read_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(base + 1), h->region_key_off, (size_t)h->n_regions + 1, d->region_key_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(base + 2), h->key_gid, h->n_keys, d->key_gid, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(base + 3), h->rec_off, n + 1, d->rec_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(base + 4), h->recs, n_slots, d->recs, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(base + 5), h->n_rec, n, d->n_rec, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(base + 6), h->read_len, n, d->read_len, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(base + 7), h->non_ambig, n, d->non_ambig, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(base + 8), h->read_flags, n, d->read_flags, 16))) return rc;
    if (h->read_id && (rc = sx_upload(ctx, sx_host_slot(base + 9), h->read_id, n, d->read_id, 16))) return rc;
    return SX_OK;
}

extern "C" int sx_link_indel_reads_dev(sx_ctx* ctx, const sx_indel_reads_sample* normal, const sx_indel_reads_sample* tumor, const sx_indel_loci* loci,
                                       sx_indel_reads_out* out_dev, uint32_t* totals_host)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    const char* what("sx_link_indel_reads_dev");
    int rc;
    if ((rc = k6b_check(ctx, what, normal, tumor, loci)) || (rc = k6b_check_out(ctx, what, out_dev))) return rc;
    sx_indel_reads_out o(*out_dev);
    return k6l_link_dev(ctx, what, SX_ST_K6B_ID, [&](unsigned* launches) { return sx_k6b_run(ctx, what, normal, tumor, loci, &o, totals_host, false, launches); });
}

extern "C" int sx_link_indel_reads(sx_ctx* ctx, const sx_indel_reads_sample* normal, const sx_indel_reads_sample* tumor, const sx_indel_loci* loci,
                                   sx_indel_reads_out* out_host, uint32_t* totals_host)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    const char* what("sx_link_indel_reads");
    int rc;
    if ((rc = k6b_check(ctx, what, normal, tumor, loci)) || (rc = k6b_check_out(ctx, what, out_host))) return rc;
    const size_t n_loci(loci->n_loci);
    if (n_loci && (!out_host->status || (out_host->cap_reads && !out_host->reads) || (out_host->cap_alts && !out_host->alts)))
        return sx_fail(ctx, SX_ERR_ARG, "%s: NULL output array", what);
    for (size_t l = 0; l < n_loci; ++l)
        if (loci->gid[l] >= loci->n_gid || (l && loci->gid[l] <= loci->gid[l - 1]))
            return sx_fail(ctx, SX_ERR_ARG, "%s: locus %zu: id %u is not ascending, or past n_gid (%u)", what, l, loci->gid[l], loci->n_gid);
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    sx_call_timer t(ctx);
    sx_indel_reads_sample dn, dt;
    sx_indel_loci dl(*loci);
    if ((rc = sx_k6b_upload_sample(ctx, what, normal, 0, loci->n_gid, &dn)) || (rc = sx_k6b_upload_sample(ctx, what, tumor, 10, loci->n_gid, &dt))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(20), loci->gid, n_loci, dl.gid, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(21), loci->gid_key, n_loci ? loci->n_gid : 0, dl.gid_key, 16))) return rc;
    // (key, is_forced_output and err_idx pass through to K5b; the link does not read them)
    sx_indel_reads_out o(*out_host);
    if ((rc = sx_take(ctx, SX_SLOT_K6B_OUT_ALT_OFF, n_loci + 1, o.alt_off, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K6B_OUT_READ_OFF, 2 * n_loci + 1, o.read_off, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K6B_OUT_STATUS, n_loci, o.status, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K6B_OUT_TOTALS, 2, o.totals, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K6B_OUT_READS, o.cap_reads, o.reads, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K6B_OUT_ALTS, o.cap_alts, o.alts, 16))) return rc;
    unsigned launches(0);
    uint32_t h_totals[2] = {0, 0};
    rc = sx_k6b_run(ctx, what, &dn, &dt, &dl, &o, h_totals, false, &launches);
    if (rc != SX_OK && rc != SX_ERR_CAPACITY) return rc;
    const int rc_run(rc);
    out_host->totals[0] = h_totals[0];
    out_host->totals[1] = h_totals[1];
    if (totals_host)
    {
        totals_host[0] = h_totals[0];
        totals_host[1] = h_totals[1];
    }
    if ((rc = sx_download(ctx, out_host->alt_off, o.alt_off, n_loci + 1))) return rc;
    if ((rc = sx_download(ctx, out_host->read_off, o.read_off, 2 * n_loci + 1))) return rc;
    if ((rc = sx_download(ctx, out_host->status, o.status, n_loci))) return rc;
    if (rc_run == SX_OK)
    {
        if ((rc = sx_download(ctx, out_host->reads, o.reads, h_totals[0]))) return rc;
        if ((rc = sx_download(ctx, out_host->alts, o.alts, h_totals[1]))) return rc;
    }
    if ((rc = t.finish(launches))) return rc;
    if ((rc = sx_check_status(ctx, what, SX_ST_K6B_ID))) return rc;
    return rc_run;
}

int sx_k6b_own_out(sx_ctx* ctx, const uint32_t n_loci, sx_indel_reads_out* o)
{
    *o = sx_indel_reads_out{};
    int rc;
    if ((rc = sx_take(ctx, SX_SLOT_K6B_OUT_ALT_OFF, (size_t)n_loci + 1, o->alt_off, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K6B_OUT_READ_OFF, 2 * (size_t)n_loci + 1, o->read_off, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K6B_OUT_STATUS, n_loci, o->status, 16))) return rc;
    return sx_take(ctx, SX_SLOT_K6B_OUT_TOTALS, 2, o->totals, 16);
}

sx_sindel_batch sx_sindel_batch_of(const sx_indel_loci* loci, const sx_indel_reads_out* o)
{
    return sx_sindel_batch{loci->n_loci, 0, loci->key, loci->is_forced_output, loci->err_idx, o->alt_off, o->alts, o->read_off, o->reads};
}

int sx_sindel_from_links_run(sx_ctx* ctx, const sx_sindel_opts* opts, const sx_indel_loci* loci, const sx_indel_reads_out* o, const double* err_prob, const uint32_t n_err,
                             sx_sindel_result* out_dev, unsigned* launches)
{
    int rc;
    const sx_sindel_batch b(sx_sindel_batch_of(loci, o));
    if ((rc = sx_k5b_run(ctx, opts, &b, err_prob, n_err, out_dev, launches))) return rc;
    const uint32_t n_loci(loci->n_loci);
    k6b_flag_results_kernel<<<std::max(1, std::min<int>((int)((n_loci + 255) / 256), ctx->sm_count * 16)), 256, 0, ctx->s_compute>>>(n_loci, o->status, out_dev);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 1;
    return SX_OK;
}

extern "C" int sx_somatic_indel_from_records_dev(sx_ctx* ctx, const sx_sindel_opts* opts, const sx_indel_reads_sample* normal, const sx_indel_reads_sample* tumor,
                                                 const sx_indel_loci* loci, const double* err_prob_host, uint32_t n_err, sx_sindel_result* out_dev)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    const char* what("sx_somatic_indel_from_records_dev");
    int rc;
    if ((rc = k6b_check(ctx, what, normal, tumor, loci))) return rc;
    if (!opts || !out_dev) return sx_fail(ctx, SX_ERR_ARG, "%s: NULL argument", what);
    if (loci->n_loci == 0) return SX_OK;
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    sx_indel_reads_out o;
    if ((rc = sx_k6b_own_out(ctx, loci->n_loci, &o))) return rc;
    if ((rc = sx_run_timed(ctx, [&](unsigned* launches) { return sx_k6b_run(ctx, what, normal, tumor, loci, &o, nullptr, true, launches); }))) return rc;
    if ((rc = sx_check_status(ctx, what, SX_ST_K6B_ID))) return rc;
    // K5b and the flags on the link's output: its checks and status word are reported as sx_somatic_indel_dev's, its time and launches added to the link's
    const sx_timing link(ctx->timing);
    ctx->timing = sx_timing{};
    const sx_sindel_batch b(sx_sindel_batch_of(loci, &o));
    if ((rc = sx_k5b_check(ctx, "sx_somatic_indel_dev", opts, &b, err_prob_host, n_err, out_dev))) return rc;
    if ((rc = sx_run_timed(ctx, [&](unsigned* launches) { return sx_sindel_from_links_run(ctx, opts, loci, &o, err_prob_host, n_err, out_dev, launches); }))) return rc;
    if ((rc = sx_check_status(ctx, "sx_somatic_indel_dev", SX_ST_SINDEL_ARG))) return rc;
    ctx->timing.kernel_ms += link.kernel_ms;
    ctx->timing.launches += link.launches;
    return SX_OK;
}
