// k6g_allele_groups.cu -- K6g allele_groups: one sample's K6 records regrouped into K5's per-group read lists, in device memory.
//
// Replaces (include/strelka_b200.h, "K6g allele_groups") what getVariantAlleleGroupGenotypeLhoodsForSample reads of the IndelBuffer:
//   starling_common/OrthogonalVariantAlleleCandidateGroupUtil.cpp:64-196   the supporting reads and their allele log-likelihoods
//   starling_common/AlleleGroupGenotype.cpp:160-180, 216-242               the exemplar entry and the contrast fold
//
// Shape of the work: every 32-byte record is read, the records of the ids some group names become 12-byte (read id, record, read) triples,
// and each supporting read becomes A+1 floats and 5 bytes -- a handful of binary searches per read, so the floor is the bytes
// (tools/germline_indel_leg.py counts them).  A CSR producer like K6b: count -> scan (sx_scan) -> write, with a sort between.
//   k6g_mark_kernel         one thread per group: the group's checks, and list_of[id] = id for every id it names (a dense table of n_gid
//                           words, as K6b's id -> locus table; several groups store the same value to one word)
//   the list builder        (k6_lists.cuh) count, scan, scatter and sort into one list per id, one warp per id in the sort; its hook
//                           (k6g_hook) marks a list that holds a read id twice (dup[id])
//   k6g_group_count_kernel  one warp per group: its status, and its supporting reads counted 32 entries of the first allele's list at a time
//                           (binary searches in the other alleles' lists)
//   scan                    of the unflagged groups' read and float counts, in place in read_off and lnp_off, -> totals; one 12-byte round
//                           trip checks the capacities
//   k6g_write_kernel        one warp per group: ploidy and the alleles' lengths, then every supporting read's A+1 floats and fields at its
//                           rank among the supporting entries (ballot + popc)
// The body is k6g_core.cuh.
#include "k6_lists.cuh"
#include "k6g_core.cuh"

namespace
{
constexpr int K6G_THREADS = 128;
constexpr int K6G_WARPS = K6G_THREADS / 32;
constexpr unsigned FULL = 0xffffffffu;

k6g_lists k6g_lists_of(const k6l_lists& L) { return k6g_lists{L.off, L.P.id, L.P.order, L.P.rec, L.P.read}; }

__global__ void k6g_mark_kernel(const sx_allele_groups G, uint32_t* __restrict__ list_of, int* __restrict__ status)
{
    bool bad(false);
    for (uint32_t g = blockIdx.x * blockDim.x + threadIdx.x; g < G.n_groups; g += gridDim.x * blockDim.x)
    {
        if (!k6g_group_ok(G, g))
        {
            bad = true;
            continue;
        }
        for (uint32_t i = G.allele_off[g]; i < G.allele_off[g + 1]; ++i) list_of[G.allele_gid[i]] = G.allele_gid[i];
        for (uint32_t i = G.contrast_off[g]; i < G.contrast_off[g + 1]; ++i) list_of[G.contrast_gid[i]] = G.contrast_gid[i];
    }
    if (bad) atomicOr(status, SX_ST_K6G_GROUP);
}

// K6g's part of the list builder's sort: dup[x] = a read id twice in id x's list
struct k6g_hook
{
    static constexpr uint32_t n_samples = 1;
    struct warp_smem
    {
    };
    uint32_t* dup;

    __device__ void begin(warp_smem&, uint32_t) const {}
    __device__ uint32_t segment(warp_smem&, uint32_t, uint32_t, uint32_t, uint32_t, const k6l_pairs&, uint32_t) const { return 0u; }
    __device__ void end(warp_smem&, const uint32_t x, const bool d, const uint32_t*, const uint32_t lane) const
    {
        if (d && lane == 0) dup[x] = 1u;
    }
};

// a group's status: SX_INDEL_READS_ST_DUP_READ when a list it names holds a read id twice
__device__ uint32_t k6g_group_status(const sx_allele_groups& G, const uint32_t g, const uint32_t* dup, const uint32_t lane)
{
    bool d(false);
    for (uint32_t i = G.allele_off[g] + lane; i < G.allele_off[g + 1]; i += 32) d |= dup[G.allele_gid[i]] != 0;
    for (uint32_t i = G.contrast_off[g] + lane; i < G.contrast_off[g + 1]; i += 32) d |= dup[G.contrast_gid[i]] != 0;
    return __any_sync(FULL, d) ? SX_INDEL_READS_ST_DUP_READ : 0u;
}

// one warp per group: status, and the counts the second scan runs over (0 for a flagged or malformed group)
__global__ void __launch_bounds__(K6G_THREADS) k6g_group_count_kernel(const sx_indel_reads_sample s, const sx_allele_groups G, const k6g_lists L, const uint32_t* __restrict__ dup,
                                                                     const sx_allele_group_reads_out o, unsigned long long* __restrict__ total_lnp)
{
    const uint32_t lane(threadIdx.x & 31), warp(threadIdx.x >> 5);
    for (uint32_t g = blockIdx.x * K6G_WARPS + warp; g < G.n_groups; g += gridDim.x * K6G_WARPS)
    {
        uint32_t st(0), n(0), A(0);
        if (k6g_group_ok(G, g)) // (a malformed group has raised SX_ST_K6G_GROUP: the call fails, its counts only need to be defined)
        {
            st = k6g_group_status(G, g, dup, lane);
            const uint32_t* agid(G.allele_gid + G.allele_off[g]);
            A = G.allele_off[g + 1] - G.allele_off[g];
            if (!st)
                for (uint32_t p0 = L.off[agid[0]]; p0 < L.off[agid[0] + 1]; p0 += 32)
                {
                    const uint32_t p(p0 + lane);
                    n += __popc(__ballot_sync(FULL, p < L.off[agid[0] + 1] && k6g_supports(s, L, agid, A, p)));
                }
        }
        if (lane == 0)
        {
            o.status[g] = st;
            o.read_off[g] = n;
            o.lnp_off[g] = n * (A + 1);
            if (n) atomicAdd(total_lnp, (unsigned long long)n * (A + 1));
        }
    }
}

__global__ void __launch_bounds__(K6G_THREADS) k6g_write_kernel(const sx_indel_reads_sample s, const sx_allele_groups G, const k6g_lists L, const sx_allele_group_reads_out o)
{
    const uint32_t lane(threadIdx.x & 31), warp(threadIdx.x >> 5);
    for (uint32_t g = blockIdx.x * K6G_WARPS + warp; g < G.n_groups; g += gridDim.x * K6G_WARPS)
    {
        if (!k6g_group_ok(G, g)) continue; // (the call fails with SX_ST_K6G_GROUP; nothing of such a group can be addressed)
        const uint32_t a0(G.allele_off[g]), A(G.allele_off[g + 1] - a0);
        const uint32_t *agid(G.allele_gid + a0), *cgid(G.contrast_gid + G.contrast_off[g]), C(G.contrast_off[g + 1] - G.contrast_off[g]);
        if (lane == 0) o.ploidy[g] = G.ploidy[g];
        if (lane < A)
        {
            o.allele_del_len[a0 + lane] = G.gid_key[agid[lane]].del_len;
            o.allele_ins_len[a0 + lane] = G.gid_key[agid[lane]].ins_len;
        }
        if (o.status[g]) continue;
        uint32_t k(o.read_off[g]);
        float* lnp(o.allele_lnp + o.lnp_off[g]);
        for (uint32_t p0 = L.off[agid[0]]; p0 < L.off[agid[0] + 1]; p0 += 32)
        {
            const uint32_t p(p0 + lane);
            const bool sup(p < L.off[agid[0] + 1] && k6g_supports(s, L, agid, A, p));
            const unsigned m(__ballot_sync(FULL, sup));
            if (sup)
            {
                const uint32_t at(k + __popc(m & ((1u << lane) - 1u)));
                float v[SX_INDEL_MAX_ALLELES + 1];
                k6g_allele_lnp(s, L, agid, A, cgid, C, L.id[p], v);
                for (uint32_t a = 0; a <= A; ++a) lnp[(size_t)(at - o.read_off[g]) * (A + 1) + a] = v[a];
                const uint32_t r(L.read[k6g_slot(L, agid[0], p)]);
                o.read_length[at] = s.read_len[r];
                o.non_ambig[at] = s.non_ambig[r];
                o.is_fwd[at] = (s.read_flags[r] & SX_SIF_FWD) ? 1 : 0;
            }
            k += __popc(m);
        }
    }
}

// a flagged group's result: all zero; every group's status to the caller's array
__global__ void k6g_flag_results_kernel(const uint32_t n_groups, const uint32_t* __restrict__ st, sx_indel_result* __restrict__ out, uint32_t* __restrict__ status_out)
{
    for (uint32_t g = blockIdx.x * blockDim.x + threadIdx.x; g < n_groups; g += gridDim.x * blockDim.x)
    {
        if (status_out) status_out[g] = st[g];
        if (!st[g]) continue;
        uint32_t* w(reinterpret_cast<uint32_t*>(out + g));
        for (uint32_t i = 0; i < sizeof(sx_indel_result) / 4; ++i) w[i] = 0u;
    }
}

int k6g_check(sx_ctx* ctx, const char* what, const sx_indel_reads_sample* sample, const sx_allele_groups* groups)
{
    int rc;
    if ((rc = sx_k6b_check_sample(ctx, what, sample))) return rc;
    if (!groups) return sx_fail(ctx, SX_ERR_ARG, "%s: NULL argument", what);
    if (groups->n_groups && (!groups->allele_off || !groups->allele_gid || !groups->contrast_off || !groups->contrast_gid || !groups->ploidy || !groups->gid_key))
        return sx_fail(ctx, SX_ERR_ARG, "%s: NULL group array", what);
    if (groups->n_groups > 0x7fffffffu) return sx_fail(ctx, SX_ERR_RANGE, "%s: more than 2^31 - 1 groups", what);
    return SX_OK;
}

int k6g_check_out(sx_ctx* ctx, const char* what, const sx_allele_group_reads_out* o, const uint32_t n_groups)
{
    if (!o || !o->read_off || !o->lnp_off || !o->allele_off || !o->totals) return sx_fail(ctx, SX_ERR_ARG, "%s: NULL output array", what);
    if (n_groups && (!o->ploidy || !o->allele_del_len || !o->allele_ins_len || !o->status)) return sx_fail(ctx, SX_ERR_ARG, "%s: NULL output array", what);
    return SX_OK;
}

// the K6g scratch and own-output slots hold a few words past every array (16 bytes), as K6b's
int k6g_take_out(sx_ctx* ctx, const uint32_t n_groups, sx_allele_group_reads_out* o)
{
    *o = sx_allele_group_reads_out{};
    const size_t n(n_groups);
    int rc;
    if ((rc = sx_take(ctx, SX_SLOT_K6G_OUT_READ_OFF, n + 1, o->read_off, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K6G_OUT_LNP_OFF, n + 1, o->lnp_off, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K6G_OUT_ALLELE_OFF, n + 1, o->allele_off, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K6G_OUT_PLOIDY, n, o->ploidy, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K6G_OUT_STATUS, n, o->status, 16))) return rc;
    return sx_take(ctx, SX_SLOT_K6G_OUT_TOTALS, 2, o->totals, 16);
}
} // namespace

int sx_k6g_run(sx_ctx* ctx, const char* what, const sx_indel_reads_sample* sample, const sx_allele_groups* groups, sx_allele_group_reads_out* o, uint32_t* totals_host,
               const bool own_out, unsigned* launches)
{
    cudaStream_t st(ctx->s_compute);
    const uint32_t n_groups(groups->n_groups), n_gid(groups->n_gid);
    int rc;
    if (n_groups == 0)
    {
        SX_CUDA(ctx, cudaMemsetAsync(o->totals, 0, 8, st));
        SX_CUDA(ctx, cudaMemsetAsync(o->read_off, 0, 4, st));
        SX_CUDA(ctx, cudaMemsetAsync(o->lnp_off, 0, 4, st));
        SX_CUDA(ctx, cudaMemsetAsync(o->allele_off, 0, 4, st));
        if (totals_host) totals_host[0] = totals_host[1] = 0;
        return SX_OK;
    }
    uint32_t *list_of(nullptr), *dup(nullptr);
    unsigned long long* lnp64(nullptr); // allele_lnp floats
    if ((rc = sx_take(ctx, SX_SLOT_K6G_LIST_OF, n_gid, list_of, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K6G_DUP, n_gid, dup, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K6G_LNP64, 1, lnp64, 0))) return rc;

    const k6b_view v(k6g_view(*sample, n_gid, list_of));
    SX_CUDA(ctx, cudaMemsetAsync(list_of, 0xFF, (size_t)n_gid * 4, st));
    SX_CUDA(ctx, cudaMemsetAsync(dup, 0, (size_t)n_gid * 4, st));
    SX_CUDA(ctx, cudaMemsetAsync(lnp64, 0, 8, st));
    k6g_mark_kernel<<<k6l_grid(ctx, n_groups, 256), 256, 0, st>>>(*groups, list_of, ctx->d_status);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 1;
    k6l_lists lists;
    if ((rc = k6l_build(ctx, what, v, n_gid, k6g_hook{dup}, &lists, launches))) return rc;
    const k6g_lists L(k6g_lists_of(lists));
    k6g_group_count_kernel<<<k6l_grid(ctx, n_groups, K6G_WARPS), K6G_THREADS, 0, st>>>(*sample, *groups, L, dup, *o, lnp64);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 1;
    SX_CUDA(ctx, cudaMemcpyAsync(o->allele_off, groups->allele_off, ((size_t)n_groups + 1) * 4, cudaMemcpyDeviceToDevice, st));
    const sx_scan_set out = {2, {{o->read_off, n_groups, SX_SCAN_EXCLUSIVE | SX_SCAN_CLOSE, o->totals}, {o->lnp_off, n_groups, SX_SCAN_EXCLUSIVE | SX_SCAN_CLOSE, o->totals + 1}}};
    if ((rc = sx_scan(ctx, SX_SLOT_K6L_SUMS, out, launches))) return rc;
    uint32_t h[3] = {0, 0, 0}; // reads, floats, alleles
    unsigned long long n_lnp64(0);
    SX_CUDA(ctx, cudaMemcpyAsync(h, o->totals, 8, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaMemcpyAsync(h + 2, o->allele_off + n_groups, 4, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaMemcpyAsync(&n_lnp64, lnp64, 8, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaStreamSynchronize(st));
    if (n_lnp64 != h[1]) return sx_fail(ctx, SX_ERR_RANGE, "%s: %llu allele log-likelihoods: the offsets are 32-bit", what, n_lnp64);
    if (totals_host)
    {
        totals_host[0] = h[0];
        totals_host[1] = h[1];
    }
    if (own_out)
    {
        if ((rc = sx_take(ctx, SX_SLOT_K6G_OUT_DEL_LEN, h[2], o->allele_del_len, 16))) return rc;
        if ((rc = sx_take(ctx, SX_SLOT_K6G_OUT_INS_LEN, h[2], o->allele_ins_len, 16))) return rc;
        if ((rc = sx_take(ctx, SX_SLOT_K6G_OUT_LNP, h[1], o->allele_lnp, 16))) return rc;
        if ((rc = sx_take(ctx, SX_SLOT_K6G_OUT_READ_LENGTH, h[0], o->read_length, 16))) return rc;
        if ((rc = sx_take(ctx, SX_SLOT_K6G_OUT_NON_AMBIG, h[0], o->non_ambig, 16))) return rc;
        if ((rc = sx_take(ctx, SX_SLOT_K6G_OUT_IS_FWD, h[0], o->is_fwd, 16))) return rc;
        o->cap_reads = h[0];
        o->cap_lnp = h[1];
    }
    if (h[0] > o->cap_reads || h[1] > o->cap_lnp)
        return sx_fail(ctx, SX_ERR_CAPACITY, "%s: output capacity too small: %u reads, %u allele log-likelihoods needed", what, h[0], h[1]);
    if ((h[0] && (!o->read_length || !o->non_ambig || !o->is_fwd)) || (h[1] && !o->allele_lnp)) return sx_fail(ctx, SX_ERR_ARG, "%s: NULL output array", what);
    k6g_write_kernel<<<k6l_grid(ctx, n_groups, K6G_WARPS), K6G_THREADS, 0, st>>>(*sample, *groups, L, *o);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 1;
    return SX_OK;
}

extern "C" int sx_link_allele_groups_dev(sx_ctx* ctx, const sx_indel_reads_sample* sample, const sx_allele_groups* groups, sx_allele_group_reads_out* out_dev,
                                         uint32_t* totals_host)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    const char* what("sx_link_allele_groups_dev");
    int rc;
    if ((rc = k6g_check(ctx, what, sample, groups)) || (rc = k6g_check_out(ctx, what, out_dev, groups->n_groups))) return rc;
    sx_allele_group_reads_out o(*out_dev);
    return k6l_link_dev(ctx, what, SX_ST_K6G_GROUP | SX_ST_K6B_ID, [&](unsigned* launches) { return sx_k6g_run(ctx, what, sample, groups, &o, totals_host, false, launches); });
}

extern "C" int sx_link_allele_groups(sx_ctx* ctx, const sx_indel_reads_sample* sample, const sx_allele_groups* groups, sx_allele_group_reads_out* out_host,
                                     uint32_t* totals_host)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    const char* what("sx_link_allele_groups");
    int rc;
    if ((rc = k6g_check(ctx, what, sample, groups)) || (rc = k6g_check_out(ctx, what, out_host, groups->n_groups))) return rc;
    const size_t n(groups->n_groups);
    for (size_t g = 0; g < n; ++g)
        if (!k6g_group_ok(*groups, (uint32_t)g))
            return sx_fail(ctx, SX_ERR_ARG, "%s: group %zu: allele count outside 1..%d, ploidy outside {1,2}, an id past n_gid (%u), or offsets that do not ascend from 0", what, g,
                           SX_INDEL_MAX_ALLELES, groups->n_gid);
    if ((out_host->cap_reads && (!out_host->read_length || !out_host->non_ambig || !out_host->is_fwd)) || (out_host->cap_lnp && !out_host->allele_lnp))
        return sx_fail(ctx, SX_ERR_ARG, "%s: NULL output array", what);
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    sx_call_timer t(ctx);
    sx_indel_reads_sample ds;
    sx_allele_groups dg(*groups);
    const size_t n_al(n ? groups->allele_off[n] : 0), n_co(n ? groups->contrast_off[n] : 0);
    if ((rc = sx_k6b_upload_sample(ctx, what, sample, 0, groups->n_gid, &ds))) return rc;
    if (n)
    {
        if ((rc = sx_upload(ctx, sx_host_slot(10), groups->allele_off, n + 1, dg.allele_off, 16))) return rc;
        if ((rc = sx_upload(ctx, sx_host_slot(11), groups->allele_gid, n_al, dg.allele_gid, 16))) return rc;
        if ((rc = sx_upload(ctx, sx_host_slot(12), groups->contrast_off, n + 1, dg.contrast_off, 16))) return rc;
        if ((rc = sx_upload(ctx, sx_host_slot(13), groups->contrast_gid, n_co, dg.contrast_gid, 16))) return rc;
        if ((rc = sx_upload(ctx, sx_host_slot(14), groups->ploidy, n, dg.ploidy, 16))) return rc;
        if ((rc = sx_upload(ctx, sx_host_slot(15), groups->gid_key, groups->n_gid, dg.gid_key, 16))) return rc;
    }
    sx_allele_group_reads_out o(*out_host);
    if ((rc = sx_take(ctx, sx_host_slot(16), n + 1, o.read_off, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(17), n + 1, o.lnp_off, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(18), n + 1, o.allele_off, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(19), n, o.ploidy, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(20), n_al, o.allele_del_len, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(21), n_al, o.allele_ins_len, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(22), o.cap_lnp, o.allele_lnp, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(23), o.cap_reads, o.read_length, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(24), o.cap_reads, o.non_ambig, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(25), o.cap_reads, o.is_fwd, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(26), n, o.status, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(27), 2, o.totals, 16))) return rc;
    unsigned launches(0);
    uint32_t h_totals[2] = {0, 0};
    rc = sx_k6g_run(ctx, what, &ds, &dg, &o, h_totals, false, &launches);
    if (rc != SX_OK && rc != SX_ERR_CAPACITY) return rc;
    const int rc_run(rc);
    out_host->totals[0] = h_totals[0];
    out_host->totals[1] = h_totals[1];
    if (totals_host)
    {
        totals_host[0] = h_totals[0];
        totals_host[1] = h_totals[1];
    }
    if ((rc = sx_download(ctx, out_host->read_off, o.read_off, n + 1))) return rc;
    if ((rc = sx_download(ctx, out_host->lnp_off, o.lnp_off, n + 1))) return rc;
    if ((rc = sx_download(ctx, out_host->allele_off, o.allele_off, n + 1))) return rc;
    if ((rc = sx_download(ctx, out_host->status, o.status, n))) return rc;
    if (rc_run == SX_OK)
    {
        if ((rc = sx_download(ctx, out_host->ploidy, o.ploidy, n))) return rc;
        if ((rc = sx_download(ctx, out_host->allele_del_len, o.allele_del_len, n_al))) return rc;
        if ((rc = sx_download(ctx, out_host->allele_ins_len, o.allele_ins_len, n_al))) return rc;
        if ((rc = sx_download(ctx, out_host->allele_lnp, o.allele_lnp, h_totals[1]))) return rc;
        if ((rc = sx_download(ctx, out_host->read_length, o.read_length, h_totals[0]))) return rc;
        if ((rc = sx_download(ctx, out_host->non_ambig, o.non_ambig, h_totals[0]))) return rc;
        if ((rc = sx_download(ctx, out_host->is_fwd, o.is_fwd, h_totals[0]))) return rc;
    }
    if ((rc = t.finish(launches))) return rc;
    if ((rc = sx_check_status(ctx, what, SX_ST_K6G_GROUP | SX_ST_K6B_ID))) return rc;
    return rc_run;
}

extern "C" int sx_indel_gl_from_records_dev(sx_ctx* ctx, const sx_indel_reads_sample* sample, const sx_allele_groups* groups, sx_indel_result* out_dev, uint32_t* status_dev)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    const char* what("sx_indel_gl_from_records_dev");
    int rc;
    if ((rc = k6g_check(ctx, what, sample, groups))) return rc;
    if (!out_dev) return sx_fail(ctx, SX_ERR_ARG, "%s: NULL argument", what);
    const uint32_t n(groups->n_groups);
    if (n == 0) return SX_OK;
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    sx_allele_group_reads_out o;
    if ((rc = k6g_take_out(ctx, n, &o))) return rc;
    if ((rc = sx_run_timed(ctx, [&](unsigned* launches) { return sx_k6g_run(ctx, what, sample, groups, &o, nullptr, true, launches); }))) return rc;
    if ((rc = sx_check_status(ctx, what, SX_ST_K6G_GROUP | SX_ST_K6B_ID))) return rc;
    // K5 and the flags on the link's output, their time and launches added to the link's
    const sx_timing link(ctx->timing);
    ctx->timing = sx_timing{};
    const sx_indel_batch b{n, o.read_off, o.lnp_off, o.allele_off, o.ploidy, o.allele_del_len, o.allele_ins_len, o.allele_lnp, o.read_length, o.non_ambig, o.is_fwd};
    rc = sx_run_timed(ctx, [&](unsigned* launches) -> int {
        int r;
        if ((r = sx_k5_run(ctx, &b, out_dev, launches))) return r;
        k6g_flag_results_kernel<<<std::max(1, std::min<int>((int)((n + 255) / 256), ctx->sm_count * 16)), 256, 0, ctx->s_compute>>>(n, o.status, out_dev, status_dev);
        SX_CUDA(ctx, cudaGetLastError());
        *launches += 1;
        return SX_OK;
    });
    if (rc) return rc;
    if ((rc = sx_check_status(ctx, "sx_indel_gl"))) return rc;
    ctx->timing.kernel_ms += link.kernel_ms;
    ctx->timing.launches += link.launches;
    return SX_OK;
}
