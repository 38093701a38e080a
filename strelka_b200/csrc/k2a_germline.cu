// k2a_germline.cu -- K2a site_gl_germline: per-site diploid genotype likelihoods, PLs and posteriors from a pileup.
//
// One warp per group of sites, two kernels:
//   k2a_germline12_kernel         twelve sites per warp: batches whose sites all hold <= K2_CAP12 (96) calls and that do not ask for the
//                                 dependent error probabilities (the whole-path pipeline's batches)
//   k2a_germline_batch_kernel<B>  B sites per warp: B = 4 for the other batches whose sites all hold <= K2_CAP_SMEM (256) calls, B = 1 for
//                                 batches with a deeper site (up to K2_CAP_BIG calls, through a global scratch)
// Both fuse, in the reference's order (paths relative to /root/reference/src/c++/lib/):
//   CleanPileupFilter              starling_common/PileupCleaner.cpp:30-64
//   adjust_joint_eprob             blt_common/adjust_joint_eprob.cpp:60-243    (dependent error probabilities)
//   get_diploid_gt_lhood x3        blt_common/position_snp_call_pprob_digt.cpp:326-385 (all / fwd-specific / rev-specific)
//   position_snp_call_pprob_digt   :471-539  (PLs, calculate_result_set for genomic and polymorphic priors, strand bias)
//
// Parity contract.  The likelihoods are float sums taken in pileup order; the integer PLs are rounded from them, so every
// float operation is reproduced in the reference's order and rounding:
//   * the 10 genotypes x {all, fwd, rev} accumulate in 30 lanes, each lane adding its terms call by call;
//   * std::log(float) / std::pow(float,float) are the glibc-FMA-variant mirrors of sx_libm_mirror.h;
//   * std::sort's permutation of each (strand x base) group is reproduced by sx_stdsort_mirror.h (one lane per group);
//   * q-only terms come from host tables (sx_context.cu).
// The posterior normalisation runs in double with CUDA's exp/log10 (<= 1 ulp from glibc's): ref_pprob is a tolerance field, and
// an integer Q derived from it can only differ if the probability sits within ~1e-15 (relative) of a rounding boundary.
#include "sx_device_util.cuh"
#include "sx_internal.h"
#include "sx_libm_mirror.h"
#include "sx_stdsort_mirror.h"

#include <algorithm>

namespace
{
constexpr int K2_WARPS = 4;
constexpr int K2_CAP_SMEM = 256;   // cleaned calls per site handled in shared memory
constexpr int K2_CAP_BIG = 8192;   // cleaned calls per site handled through the global scratch
constexpr unsigned FULL = 0xffffffffu;

struct germ_tables // the slice of sx_tables this kernel reads, staged in shared memory
{
    float eprob[SX_MAX_QSCORE + 1], val1[SX_MAX_QSCORE + 1], val2[SX_MAX_QSCORE + 1], weight[SX_MAX_QSCORE + 1], depmin[SX_MAX_QSCORE + 1];
    float lnprior[2][5][2][10];
};

struct QKey // sort_icall_by_eprob's view: quality of call index i
{
    const uint16_t* calls;
    __device__ __forceinline__ uint32_t operator[](uint32_t i) const { return calls[i] & 63u; }
};

struct PKey // the same for elements that carry their quality: (q << 7) | call index (the twelve-site kernel: one shared load less per comparison)
{
    __device__ __forceinline__ uint32_t operator[](uint32_t packed) const { return packed >> 7; }
};

__device__ __forceinline__ float dependent_eprob(float eprob, float vexp) // get_dependent_eprob, adjust_joint_eprob.cpp:60-70
{
    const float val = sx_powf(eprob, vexp);
    const float frac = f_div(f_sub(1.0f, val), f_sub(1.0f, eprob));
    const float x = f_add(f_mul(frac, val), f_mul(f_sub(1.0f, frac), 0.75f));
    return (eprob < x) ? x : eprob; // std::max(eprob, x)
}

// (1-mismatch_frac)*opt.bsnp_ssd_no_mismatch + mismatch_frac*opt.bsnp_ssd_one_mismatch : float*double, summed in double, narrowed
__device__ __forceinline__ float vexp_frac_of(float mismatch_frac, double ssd_no, double ssd_one)
{
    return static_cast<float>(d_add(d_mul(static_cast<double>(f_sub(1.0f, mismatch_frac)), ssd_no), d_mul(static_cast<double>(mismatch_frac), ssd_one)));
}

// expect2(obs, gt) for obs 0..3 packed 2 bits each  (blt_util/digt.hh:119-140)
__device__ __forceinline__ uint32_t expect2_pack(uint32_t gt)
{
    if (gt < 4) return 2u << (2 * gt);
    const uint32_t a = (gt < 7) ? 0u : (gt < 9) ? 1u : 2u;
    const uint32_t b = (gt < 7) ? gt - 3u : (gt < 9) ? gt - 5u : 3u;
    return (1u << (2 * a)) | (1u << (2 * b));
}

// the genotype priors into a kernel's shared-memory tables
__device__ __forceinline__ void stage_lnprior(float (*dst)[5][2][10], const sx_tables* __restrict__ tables)
{
    for (int i = threadIdx.x; i < 200; i += blockDim.x) (&dst[0][0][0][0])[i] = (&tables->g_lnprior[0][0][0][0])[i];
}

struct rs_out
{
    double ref_pprob;
    uint32_t max_gt;
    int snp_qphred, max_gt_qphred;
};

// calculate_result_set (position_snp_call_pprob_digt.cpp:412-433) + normalizeLogDistro/prob_comp (blt_util/prob_util.hh:179-237).
// lanes 0..9 hold lhood[gt]; all lanes return the same result.
__device__ __forceinline__ rs_out result_set(float lh, const float* lnprior, uint32_t ref_gt, uint32_t lane)
{
    const double pp = (lane < 10) ? static_cast<double>(f_add(lh, lnprior[lane])) : 0.0;
    // first maximum, strict '>' scan
    double mx = shfl_d(pp, 0);
    uint32_t max_gt = 0;
#pragma unroll
    for (int gt = 1; gt < 10; ++gt)
    {
        const double v = shfl_d(pp, gt);
        if (v > mx)
        {
            mx = v;
            max_gt = gt;
        }
    }
    const double e = (lane < 10) ? sx_exp(d_sub(pp, mx)) : 0.0;
    double sum = 0.0;
#pragma unroll
    for (int gt = 0; gt < 10; ++gt) sum = d_add(sum, shfl_d(e, gt));
    sum = d_div(1.0, sum);
    const double p = d_mul(e, sum);
    double comp = 0.0;
#pragma unroll
    for (int gt = 0; gt < 10; ++gt)
    {
        const double v = shfl_d(p, gt);
        if (gt != (int)max_gt) comp = d_add(comp, v);
    }
    rs_out o;
    o.max_gt = max_gt;
    o.ref_pprob = shfl_d(p, ref_gt);
    o.snp_qphred = error_prob_to_qphred_d(o.ref_pprob);
    o.max_gt_qphred = error_prob_to_qphred_d(comp);
    return o;
}

// ------------------------------------------------------------------------------------------------------------------
// Warp-wide steps of one site in k2a_germline_batch_kernel.  w_calls / w_val / w_ord are the site's cleaned calls, their values and
// the per-group order of call indices.

// CleanPileupFilter: the calls with is_call_filter == 0 to w_calls, order kept.  Returns their count; `nonref` (warp-uniform): one of
// them is not the reference base.
__device__ __forceinline__ uint32_t clean_pileup(const uint16_t* __restrict__ calls, uint32_t c0, uint32_t n_raw, uint32_t ref_gt, uint16_t* w_calls, uint32_t lane, bool& nonref)
{
    uint32_t n = 0;
    nonref = false;
    for (uint32_t b = 0; b < n_raw; b += 32)
    {
        const uint32_t i = b + lane;
        const uint32_t c = i < n_raw ? calls[c0 + i] : 0x1000u;
        const bool keep = !((c >> 12) & 1u);
        const uint32_t m = __ballot_sync(FULL, keep);
        if (keep)
        {
            w_calls[n + __popc(m & ((1u << lane) - 1u))] = static_cast<uint16_t>(c);
            if (((c >> 6) & 15u) != ref_gt) nonref = true;
        }
        n += __popc(m);
    }
    nonref = __any_sync(FULL, nonref);
    __syncwarp();
    return n;
}

// adjust_joint_eprob's groups, is_fwd + 2*base_id over the calls with q >= 3: a stable partition of the call indices into w_ord,
// group g at [gstart[g], gstart[g + 1])
__device__ __forceinline__ void partition_groups(const uint16_t* w_calls, uint32_t n, uint16_t* w_ord, uint32_t* gstart, uint32_t lane)
{
    uint32_t start = 0;
    for (uint32_t g = 0; g < 8; ++g)
    {
        if (lane == 0) gstart[g] = start;
        for (uint32_t b = 0; b < n; b += 32)
        {
            const uint32_t i = b + lane;
            bool in = false;
            if (i < n)
            {
                const uint32_t c = w_calls[i];
                in = ((c & 63u) >= 3u) && ((((c >> 10) & 1u) + 2u * ((c >> 6) & 15u)) == g);
            }
            const uint32_t m = __ballot_sync(FULL, in);
            if (in) w_ord[start + __popc(m & ((1u << lane) - 1u))] = static_cast<uint16_t>(i);
            start += __popc(m);
        }
    }
    if (lane == 0) gstart[8] = start;
}

// the warp's region of the global scratch, for a site deeper than the shared-memory tile (B = 1 only: one region per warp)
__device__ __forceinline__ void to_scratch(unsigned char* scratch, uint32_t gwarp, uint16_t*& w_calls, float*& w_val, uint16_t*& w_ord)
{
    unsigned char* r = scratch + (size_t)gwarp * (K2_CAP_BIG * 8);
    w_calls = reinterpret_cast<uint16_t*>(r);
    w_ord = reinterpret_cast<uint16_t*>(r + K2_CAP_BIG * 2);
    w_val = reinterpret_cast<float*>(r + K2_CAP_BIG * 4);
}

// ------------------------------------------------------------------------------------------------------------------
// B sites per warp.  The per-group phase of adjust_joint_eprob (weight sums in pileup order, the std::sort mirror, the exponent
// chain) is serial per (strand x base) group.  Phase A (filter, grouping) and phase C (logf, likelihoods, posteriors) run warp-wide,
// site after site; phase B runs once for the 8 * B (site, group) pairs, one per lane, so B = 4 keeps all 32 lanes on it.
//   B = 4: every site holds <= cap calls, cap = the deepest site rounded up to 32 (a shallow batch leaves room for more resident CTAs).
//   B = 1: cap = K2_CAP_SMEM; a deeper site takes the warp's K2_CAP_BIG-call region of `scratch` instead of its shared-memory tile.
//          Only this layout takes deep sites, so a warp needs one such region, not B, and the B = 4 code has no scratch path.
// A site over cap without a scratch region cannot reach the kernel (the host checks the deepest site); it would set status bit 16
// and count as empty.  Phases B and C are written out here rather than as device functions: B = 4 then compiles to the same SASS
// as the four-site kernel this template replaced, which the helper-function form did not (it ran about 1 % slower).
// ------------------------------------------------------------------------------------------------------------------
constexpr int K2_BATCH = 4;

template <int B>
__global__ void __launch_bounds__(K2_WARPS * 32) k2a_germline_batch_kernel(const uint32_t* __restrict__ site_off, const uint16_t* __restrict__ calls_g,
                                                                           const char* __restrict__ ref_base, const uint8_t* __restrict__ ploidy,
                                                                           uint32_t n_sites, int is_always_test, const sx_tables* __restrict__ tables,
                                                                           sx_digt_result* __restrict__ out, uint32_t* __restrict__ de_off,
                                                                           float* __restrict__ de_out, int* __restrict__ status, uint32_t cap,
                                                                           unsigned char* __restrict__ scratch)
{
    __shared__ germ_tables T;
    // per (warp, site slot): `cap` cleaned calls (uint16), their values (float), the per-group order (uint16)
    extern __shared__ __align__(16) unsigned char k2_dyn[];
    float* const s_val_all = reinterpret_cast<float*>(k2_dyn);
    uint16_t* const s_calls_all = reinterpret_cast<uint16_t*>(k2_dyn + (size_t)K2_WARPS * B * cap * 4);
    uint16_t* const s_ord_all = s_calls_all + (size_t)K2_WARPS * B * cap;
    __shared__ uint32_t s_gstart[K2_WARPS][B][9];
    __shared__ uint32_t s_n[K2_WARPS][B];
    for (int i = threadIdx.x; i <= SX_MAX_QSCORE; i += blockDim.x)
    {
        T.eprob[i] = tables->g_eprob[i];
        T.val1[i] = tables->g_val1[i];
        T.val2[i] = tables->g_val2[i];
        T.weight[i] = tables->g_weight[i];
        T.depmin[i] = tables->g_depmin[i];
    }
    stage_lnprior(T.lnprior, tables);
    __syncthreads();
    const float log_one_third = tables->g_log_one_third;
    const float ln10f = tables->g_ln10f;
    const float min_vexp = tables->g_min_vexp;
    const double ssd_no = tables->g_ssd_no_mismatch, ssd_one = tables->g_ssd_one_mismatch;
    const bool is_dep = tables->g_is_dependent_eprob != 0;
    const bool is_limit_vexp = tables->g_is_min_vexp != 0;

    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t gwarp = blockIdx.x * K2_WARPS + warp, nwarps = gridDim.x * K2_WARPS;

    for (uint32_t base = gwarp * B; base < n_sites; base += nwarps * B)
    {
        const uint32_t nb = min((uint32_t)B, n_sites - base);
        // ---- phase A, site by site: CleanPileupFilter, initial eprobs, grouping
        uint32_t nonref_mask = 0;
        bool deep = false; // (B = 1) the site holds more than cap calls: its arrays are in the scratch
        for (uint32_t s = 0; s < B; ++s)
        {
            uint16_t* w_calls = s_calls_all + (warp * B + s) * cap;
            float* w_val = s_val_all + (warp * B + s) * cap;
            uint16_t* w_ord = s_ord_all + (warp * B + s) * cap;
            uint32_t n = 0;
            bool nonref = false;
            if (s < nb)
            {
                const uint32_t site = base + s;
                const uint32_t c0 = site_off[site], c1 = site_off[site + 1];
                uint32_t n_raw = c1 - c0;
                if (n_raw > cap)
                {
                    deep = B == 1 && scratch != nullptr && n_raw <= K2_CAP_BIG;
                    if (deep)
                    {
                        to_scratch(scratch, gwarp, w_calls, w_val, w_ord);
                    }
                    else
                    {
                        if (lane == 0) atomicOr(status, SX_ST_SITE_DEPTH);
                        n_raw = 0;
                    }
                }
                const char rb = ref_base[site];
                const uint32_t ref_gt = rb == 'A' ? 0u : rb == 'C' ? 1u : rb == 'G' ? 2u : rb == 'T' ? 3u : 4u;
                n = clean_pileup(calls_g, c0, n_raw, ref_gt, w_calls, lane, nonref);
                for (uint32_t i = lane; i < n; i += 32) w_val[i] = T.eprob[w_calls[i] & 63u];
            }
            if (nonref) nonref_mask |= 1u << s;
            if (lane == 0) s_n[warp][s] = n;
            if (is_dep) partition_groups(w_calls, n, w_ord, s_gstart[warp][s], lane);
        }
        __syncwarp();
        // ---- phase B: one (site, group) pair per lane -- adjust_icalls_eprob (adjust_joint_eprob.cpp:100-180)
        if (is_dep && lane < 8 * B)
        {
            const uint32_t s = lane >> 3, g = lane & 7u;
            uint16_t* w_calls = s_calls_all + (warp * B + s) * cap;
            float* w_val = s_val_all + (warp * B + s) * cap;
            uint16_t* w_ord = s_ord_all + (warp * B + s) * cap;
            if (deep) to_scratch(scratch, gwarp, w_calls, w_val, w_ord);
            const uint32_t g0 = s_gstart[warp][s][g], sz = s_gstart[warp][s][g + 1] - g0;
            if (sz)
            {
                uint16_t* ic = w_ord + g0;
                float num = 0.f, den = 0.f; // :112-127, in pileup order (before the sort)
                for (uint32_t k = 0; k < sz; ++k)
                {
                    const uint32_t c = w_calls[ic[k]];
                    const float weight = T.weight[c & 63u];
                    den = f_add(den, weight);
                    if ((c >> 11) & 1u) num = f_add(num, weight);
                }
                float mismatch_frac = 0.f;
                if (static_cast<double>(den) > 0.) mismatch_frac = f_div(num, den);
                const float vexp_frac = vexp_frac_of(mismatch_frac, ssd_no, ssd_one);
                const QKey key{w_calls};
                sx_stdsort_desc(ic, sz, key);
                float vexp = 1.0f;
                bool is_min_vexp = false;
                const float step = f_sub(1.0f, vexp_frac);
                for (uint32_t k = 0; k < sz; ++k)
                {
                    const uint32_t idx = ic[k];
                    const uint32_t q = w_calls[idx] & 63u;
                    if (!is_min_vexp)
                    {
                        w_val[idx] = dependent_eprob(T.eprob[q], vexp);
                        const float next_vexp = f_mul(vexp, step);
                        if (is_limit_vexp)
                        {
                            is_min_vexp = (next_vexp <= min_vexp);
                            vexp = (min_vexp < next_vexp) ? next_vexp : min_vexp; // std::max(min_vexp, next_vexp)
                        }
                        else
                        {
                            vexp = next_vexp;
                        }
                    }
                    else
                    {
                        w_val[idx] = T.depmin[q]; // dependent_prob_cache: get_dependent_eprob(q, min_vexp)
                    }
                }
            }
        }
        __syncwarp();
        // ---- phase C, site by site: likelihoods and posteriors
        for (uint32_t s = 0; s < nb; ++s)
        {
            const uint32_t site = base + s;
            uint16_t* w_calls = s_calls_all + (warp * B + s) * cap;
            float* w_val = s_val_all + (warp * B + s) * cap;
            uint16_t* w_ord = s_ord_all + (warp * B + s) * cap;
            if (deep) to_scratch(scratch, gwarp, w_calls, w_val, w_ord);
            const uint32_t n = s_n[warp][s];
            const bool nonref = (nonref_mask >> s) & 1u;
            const char rb = ref_base[site];
            const uint32_t ref_gt = rb == 'A' ? 0u : rb == 'C' ? 1u : rb == 'G' ? 2u : rb == 'T' ? 3u : 4u;
            if (de_out != nullptr)
            {
                const uint32_t o = de_off[site];
                for (uint32_t i = lane; i < n; i += 32) de_out[o + i] = w_val[i];
                __syncwarp();
                if (out == nullptr) continue;
            }
            sx_digt_result* res = out + site;
            const bool computed = (ref_gt < 4u) && (is_always_test || nonref);
            if (!computed) // diploid_genotype::reset() values
            {
                uint32_t* w = reinterpret_cast<uint32_t*>(res);
                for (uint32_t i = lane; i < sizeof(sx_digt_result) / 4; i += 32) w[i] = 0u;
                __syncwarp();
                if (lane == 0)
                {
                    res->ref_gt = (ref_gt < 4u) ? ref_gt : 0u;
                    res->n_used_calls = n;
                }
                continue;
            }
            // val[0] = std::log(eprob) + log_one_third for every call (position_snp_call_pprob_digt.cpp:352)
            for (uint32_t i = lane; i < n; i += 32) w_val[i] = f_add(sx_logf(w_val[i]), log_one_third);
            __syncwarp();
            // get_diploid_gt_lhood: lanes 0-9 all calls, 10-19 fwd-strand-specific, 20-29 rev-strand-specific
            const uint32_t pass = lane / 10u, gt = lane - pass * 10u;
            const uint32_t e2_gt = expect2_pack(gt < 10u ? gt : 0u), e2_ref = expect2_pack(ref_gt);
            float lh = 0.f;
            if (lane < 30)
            {
                for (uint32_t i = 0; i < n; ++i)
                {
                    const uint32_t c = w_calls[i];
                    const uint32_t q = c & 63u, obs = (c >> 6) & 3u, fwd = (c >> 10) & 1u;
                    const bool force_ref = (pass != 0u) && ((pass == 1u) != (fwd != 0u));
                    const uint32_t k = ((force_ref ? e2_ref : e2_gt) >> (2u * obs)) & 3u;
                    const float v = (k == 0u) ? w_val[i] : (k == 1u) ? T.val1[q] : T.val2[q];
                    lh = f_add(lh, v);
                }
            }
            const bool haploid = ploidy != nullptr && ploidy[site] == 1;
            const uint32_t gtcount = haploid ? 4u : 10u;
            float lmax = __shfl_sync(FULL, lh, 0);
            for (uint32_t g = 1; g < gtcount; ++g)
            {
                const float v = __shfl_sync(FULL, lh, g);
                if (v > lmax) lmax = v;
            }
            uint32_t pl = 0;
            if (lane < gtcount) pl = static_cast<uint32_t>(ln_error_prob_to_qphred_f(f_sub(lh, lmax), ln10f));
            const float* pri = T.lnprior[haploid ? 1 : 0][ref_gt][0];
            const rs_out genome = result_set(lh, pri, ref_gt, lane);
            const rs_out poly = result_set(lh, pri + 10, ref_gt, lane);
            double strand_bias = 0.0;
            {
                const uint32_t tgt = genome.max_gt;
                const float lf = __shfl_sync(FULL, lh, 10 + tgt), lr = __shfl_sync(FULL, lh, 20 + tgt), l0 = __shfl_sync(FULL, lh, tgt);
                if (genome.snp_qphred != 0) strand_bias = static_cast<double>(f_sub((lf < lr) ? lr : lf, l0));
            }
            if (lane < 10)
            {
                res->lhood[lane] = lh;
                res->phredLoghood[lane] = pl;
            }
            if (lane == 0)
            {
                res->genome.ref_pprob = genome.ref_pprob;
                res->genome.max_gt = genome.max_gt;
                res->genome.snp_qphred = genome.snp_qphred;
                res->genome.max_gt_qphred = genome.max_gt_qphred;
                res->genome.pad = 0;
                res->poly.ref_pprob = poly.ref_pprob;
                res->poly.max_gt = poly.max_gt;
                res->poly.snp_qphred = poly.snp_qphred;
                res->poly.max_gt_qphred = poly.max_gt_qphred;
                res->poly.pad = 0;
                res->strand_bias = strand_bias;
                res->ref_gt = ref_gt;
                res->is_computed = 1;
                res->n_used_calls = n;
                res->pad = 0;
            }
            __syncwarp();
        }
        __syncwarp();
    }
}

// ------------------------------------------------------------------------------------------------------------------
// Twelve sites per warp.  At the whole-path pipeline's sites (every position of a ~30x contig, nearly all of them homozygous reference)
// the B-site layout leaves most lanes idle:
//   * the two posterior blocks (calculate_result_set for the genomic and the polymorphic prior) each run on 10 lanes,
//     one after the other, with the double log10 / exp sequences issued warp-wide;
//   * the likelihood accumulation keeps 30 lanes busy with all / fwd-specific / rev-specific sums although the strand-specific
//     sums are read only at SNP sites (position_snp_call_pprob_digt.cpp:522-533) and only for ONE genotype;
//   * the (strand x base) grouping takes 8 ballot rounds per site, each a loop over the calls;
//   * the serial per-group phase has 32 (site, group) lanes, of which a homozygous site fills 2 of its 8.
// Here the same arithmetic is laid out so that the lanes are full:
//   * filter and grouping: the batch's 12 sites own one contiguous call block, copied once into shared memory and taken 32 calls at a
//     time across site boundaries (a site's calls are a contiguous lane range of a chunk), three bit-plane ballots give every call its
//     (site, group) members and rank, one scan per batch the group starts;
//   * the serial phase takes a compacted list of the NON-EMPTY (site, group) pairs of 12 sites, one pair per lane;
//   * accumulation and posteriors run for THREE sites at once, 10 lanes each (lanes 30, 31 idle): the `all' sums only; the two
//     strand-specific sums of the called genotype are computed by two lanes, for SNP sites only.
// Every float sum keeps its order (one lane adds a genotype's terms call by call), so results are bit-identical to the B-site kernel's.
// ------------------------------------------------------------------------------------------------------------------
constexpr int K2_B12 = 12;

// shared-memory loads through 32-bit shared addresses: the accumulation picks one of three arrays per (call, genotype), and a selected
// C++ pointer made the compiler branch per array (cuobjdump: BSSY / BRA around every load, 16 of 32 lanes active)
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ float lds_f32(uint32_t a)
{
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t lds_u16(uint32_t a)
{
    uint16_t v;
    asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(a) : "memory");
    return v;
}
// the twelve-site kernel's view of a call, written where the call is compacted:
//   obs << 14 | (base_id >= 4) << 10 | neighbour mismatch << 9 | q << 3 | fwd
// (q << 3 is the byte offset of the call's {val1, val2} pair; phase C reads bits 3-8 and 13-15 only, and bit 13 is zero)
__device__ __forceinline__ uint32_t k2_repack(uint32_t c)
{
    return (((c >> 6) & 3u) << 14) | ((((c >> 6) & 15u) >= 4u) ? 0x400u : 0u) | (((c >> 11) & 1u) << 9) | ((c & 63u) << 3) | ((c >> 10) & 1u);
}
// adjust_joint_eprob's group of a repacked call: is_fwd + 2*base_id for q >= 3 and base_id < 4, else 0xff (not in any group)
__device__ __forceinline__ uint32_t k2_group(uint32_t r) { return (((r >> 3) & 63u) >= 3u && !(r & 0x400u)) ? (r & 1u) | ((r >> 13) & 6u) : 0xffu; }
// the lanes of elements [beg, end) in the 32-element chunk starting at element b
__device__ __forceinline__ uint32_t k2_lanes(uint32_t beg, uint32_t end, uint32_t b)
{
    const uint32_t lo = beg > b ? beg - b : 0u, hi = end > b ? end - b : 0u;
    if (lo >= 32u || hi <= lo) return 0u;
    return (hi >= 32u ? FULL : (1u << hi) - 1u) & (FULL << lo);
}
// the site of element b + lane of a twelve-site block: lane k <= 12 holds the block offset of site k's first element (lanes from the batch's
// last site + 1 on: the block's end), so the site is the number of sites 1..12 that start at or before the element.  The sites starting
// inside the chunk (about one per chunk) are taken one by one.
__device__ __forceinline__ uint32_t k2_site_of(uint32_t my_off, uint32_t b, uint32_t lane)
{
    const bool bnd = lane - 1u < 12u;
    uint32_t s = __popc(__ballot_sync(FULL, bnd && my_off <= b));
    uint32_t inner = __ballot_sync(FULL, bnd && my_off > b && my_off < b + 32u);
    while (inner)
    {
        const uint32_t o = __shfl_sync(FULL, my_off, __ffs(inner) - 1);
        inner &= inner - 1u;
        if (b + lane >= o) ++s;
    }
    return s;
}
constexpr int K2_CAP12 = 96;       // deepest site this kernel takes (shared memory: 12 sites x cap x 8 bytes per warp)
constexpr int K2_SORT_STACK12 = 16; // sx_stdsort_desc's stack for groups of at most K2_CAP12 members: 2*floor(log2(96)) + 1 = 13 entries

struct germ12_tables // the twelve-site kernel's slice of sx_tables, in shared memory
{
    float eprob[SX_MAX_QSCORE + 1], weight[SX_MAX_QSCORE + 1], val0_plain[SX_MAX_QSCORE + 1], val0_min[SX_MAX_QSCORE + 1];
    float val0_clean[SX_K2_CLEAN_RANKS][SX_MAX_QSCORE + 1];
    float lnprior[2][5][2][10];
};

// the g_val0_* rows of sx_tables (sx_internal.h), from the same device functions and operands the kernels use
__global__ void k2a_init_tables_kernel(sx_tables* __restrict__ t)
{
    const uint32_t q = threadIdx.x;
    const float log_one_third = t->g_log_one_third;
    // the exponent chain of adjust_icalls_eprob (adjust_joint_eprob.cpp:150-180) for a group whose mismatch_frac is 0
    const float step = f_sub(1.0f, vexp_frac_of(0.f, t->g_ssd_no_mismatch, t->g_ssd_one_mismatch));
    const float min_vexp = t->g_min_vexp;
    float vexp = 1.0f;
    int ranks = 0;
    bool clamped = false;
    for (int k = 0; k < SX_K2_CLEAN_RANKS && !clamped; ++k)
    {
        if (q <= SX_MAX_QSCORE) t->g_val0_clean[k][q] = f_add(sx_logf(dependent_eprob(t->g_eprob[q], vexp)), log_one_third);
        ++ranks;
        const float next_vexp = f_mul(vexp, step);
        clamped = (next_vexp <= min_vexp);
        vexp = (min_vexp < next_vexp) ? next_vexp : min_vexp;
    }
    if (q <= SX_MAX_QSCORE)
    {
        t->g_val0_plain[q] = f_add(sx_logf(t->g_eprob[q]), log_one_third);
        t->g_val0_min[q] = f_add(sx_logf(t->g_depmin[q]), log_one_third);
    }
    if (q == 0)
    {
        t->g_clean_ranks = ranks;
        t->g_clean_ok = (t->g_is_dependent_eprob && t->g_is_min_vexp && clamped) ? 1 : 0;
    }
}

__global__ void __launch_bounds__(K2_WARPS * 32, 8) k2a_germline12_kernel(const uint32_t* __restrict__ site_off, const uint16_t* __restrict__ calls_g,
                                                                       const char* __restrict__ ref_base, const uint8_t* __restrict__ ploidy,
                                                                       uint32_t n_sites, int is_always_test, const sx_tables* __restrict__ tables,
                                                                       sx_digt_result* __restrict__ out, int* __restrict__ status, uint32_t cap,
                                                                       uint32_t ord_stride)
{
    __shared__ germ12_tables T;
    // per warp: 12 sites x `cap` cleaned calls (uint16) and their values (float); an `ord_stride`-slot region (uint16) that first holds the
    // batch's raw calls as staged from global memory, then site s's per-group order at s * cap
    extern __shared__ __align__(16) unsigned char k2_dyn[];
    float* const s_val_all = reinterpret_cast<float*>(k2_dyn);
    uint16_t* const s_calls_all = reinterpret_cast<uint16_t*>(k2_dyn + (size_t)K2_WARPS * K2_B12 * cap * 4);
    uint16_t* const s_ord_all = s_calls_all + (size_t)K2_WARPS * K2_B12 * cap;
    __shared__ uint16_t s_gstart[K2_WARPS][K2_B12][10];
    __shared__ uint16_t s_n[K2_WARPS][K2_B12];
    __shared__ uint8_t s_pair[K2_WARPS][K2_B12 * 8]; // site * 8 + group, | 0x80 if the group holds a neighbour-mismatch call
    // ln P(column | genotype) of the batch's sites, phase C -> phase D; in phase A the running member count of each (site, group),
    // site * 8 + group, | 0x80 once a member carries the neighbour-mismatch bit
    __shared__ union
    {
        float lh[K2_B12][10];
        uint32_t gcnt4[K2_B12 * 2];
        uint8_t gcnt[K2_B12 * 8];
    } s_ab[K2_WARPS];
    __shared__ float s_val12[2 * (SX_MAX_QSCORE + 1)]; // {val1[q], val2[q]} side by side: the two tables no longer share a bank
    for (int i = threadIdx.x; i <= SX_MAX_QSCORE; i += blockDim.x)
    {
        T.eprob[i] = tables->g_eprob[i];
        s_val12[2 * i] = tables->g_val1[i];
        s_val12[2 * i + 1] = tables->g_val2[i];
        T.weight[i] = tables->g_weight[i];
        T.val0_plain[i] = tables->g_val0_plain[i];
        T.val0_min[i] = tables->g_val0_min[i];
    }
    for (int i = threadIdx.x; i < SX_K2_CLEAN_RANKS * (SX_MAX_QSCORE + 1); i += blockDim.x) (&T.val0_clean[0][0])[i] = (&tables->g_val0_clean[0][0])[i];
    stage_lnprior(T.lnprior, tables);
    __syncthreads();
    const float log_one_third = tables->g_log_one_third;
    const float ln10f = tables->g_ln10f;
    const float min_vexp = tables->g_min_vexp;
    const double ssd_no = tables->g_ssd_no_mismatch, ssd_one = tables->g_ssd_one_mismatch;
    const bool is_dep = tables->g_is_dependent_eprob != 0;
    const bool is_limit_vexp = tables->g_is_min_vexp != 0;
    const bool clean_ok = tables->g_clean_ok != 0;
    const uint32_t clean_ranks = static_cast<uint32_t>(tables->g_clean_ranks);

    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t lt_mask = (1u << lane) - 1u;
    const uint32_t gwarp = blockIdx.x * K2_WARPS + warp, nwarps = gridDim.x * K2_WARPS;
    const uint32_t sub = lane < 30 ? lane / 10u : 2u, sl = lane - 10u * sub, sbase = 10u * sub; // the three 10-lane blocks of phase C

    for (uint32_t base = gwarp * K2_B12; base < n_sites; base += nwarps * K2_B12)
    {
        const uint32_t nb = min((uint32_t)K2_B12, n_sites - base);
        uint32_t n_pairs = 0;
        float* const w_val0 = s_val_all + warp * K2_B12 * cap;
        uint16_t* const w_calls0 = s_calls_all + warp * K2_B12 * cap;
        uint16_t* const w_ord0 = s_ord_all + warp * ord_stride;
        // ---- phase A over the batch's call block [site_off[base], site_off[base + nb]), 32 calls at a time across site boundaries.
        //      Lane k <= 12 holds site k's block offset (from nb on: the block's end); lane k < nb the site's reference genotype (0-4, bit 0-2),
        //      haploid (bit 3) and "deeper than cap" (bit 4: status bit, and the site counts as empty).
        uint32_t my_off = site_off[base + min(lane, nb)];
        uint32_t my_info = 0;
        if (lane < nb)
        {
            const char rb = ref_base[base + lane];
            my_info = (rb == 'A' ? 0u : rb == 'C' ? 1u : rb == 'G' ? 2u : rb == 'T' ? 3u : 4u) | ((ploidy != nullptr && ploidy[base + lane] == 1) ? 8u : 0u);
        }
        const uint32_t blk0 = __shfl_sync(FULL, my_off, 0);
        my_off -= blk0;
        const uint32_t n_blk = __shfl_sync(FULL, my_off, 12);
        const uint32_t next_off = __shfl_down_sync(FULL, my_off, 1); // lane k < 12: site k's end
        if (lane < nb && next_off - my_off > cap) // the host sizes cap from the deepest site
        {
            atomicOr(status, SX_ST_SITE_DEPTH);
            my_info |= 16u;
        }
        // the raw block into the warp's order region: 16-byte loads from the 16-byte boundary at or below its first call, two in flight per lane
        // (the host sizes ord_stride from the largest block; the last 16 bytes may run past the array's end, inside its allocation's granule)
        {
            const uintptr_t a = reinterpret_cast<uintptr_t>(calls_g + blk0);
            const uint4* __restrict__ src = reinterpret_cast<const uint4*>(a & ~static_cast<uintptr_t>(15));
            uint4* const dst = reinterpret_cast<uint4*>(w_ord0);
            const uint32_t n_vec = (static_cast<uint32_t>(a & 15u) / 2u + n_blk + 7u) / 8u;
            for (uint32_t v = lane; v < n_vec; v += 64)
            {
                const uint4 x = src[v];
                uint4 y;
                if (v + 32u < n_vec) y = src[v + 32u];
                dst[v] = x;
                if (v + 32u < n_vec) dst[v + 32u] = y;
            }
        }
        if (lane < 24) s_ab[warp].gcnt4[lane] = 0u;
        __syncwarp();
        const uint16_t* const stg = w_ord0 + (reinterpret_cast<uintptr_t>(calls_g + blk0) & 15u) / 2u;
        // pass 1: CleanPileupFilter (the kept calls of site s, repacked, at w_calls[s * cap + k] in pileup order), val0_plain[q] as their value,
        // nonref per site; with the dependent model each grouped call's rank in its (site, group), in pileup order, from the three bit-plane
        // ballots of the group id ANDed with the site's lanes and the count of earlier chunks.  A grouped call's value slot holds its rank
        // until pass 2; phase B gives every grouped call its value.
        uint32_t my_cnt = 0; // lane k < 12: kept calls of site k so far
        bool my_nonref = false;
        for (uint32_t b = 0; b < n_blk; b += 32)
        {
            const uint32_t j = b + lane;
            const uint32_t s = k2_site_of(my_off, b, lane);
            const uint32_t site_m = k2_lanes(__shfl_sync(FULL, my_off, s), __shfl_sync(FULL, my_off, s + 1u), b);
            const uint32_t info = __shfl_sync(FULL, my_info, s);
            const uint32_t c = j < n_blk ? stg[j] : 0x1000u;
            const bool keep = !((c >> 12) & 1u) && !(info & 16u);
            const uint32_t km = __ballot_sync(FULL, keep);
            const uint32_t nrm = __ballot_sync(FULL, keep && ((c >> 6) & 15u) != (info & 7u));
            const uint32_t at = s * cap + __shfl_sync(FULL, my_cnt, s) + __popc(km & site_m & lt_mask);
            const uint32_t r = k2_repack(c);
            if (keep) w_calls0[at] = static_cast<uint16_t>(r);
            const uint32_t mine = k2_lanes(my_off, next_off, b); // lane k < 12: site k's lanes in this chunk
            my_cnt += __popc(km & mine);
            my_nonref = my_nonref || (nrm & mine) != 0u;
            uint32_t gi = 0xffu;
            if (is_dep)
            {
                gi = keep ? k2_group(r) : 0xffu;
                const uint32_t v = __ballot_sync(FULL, gi < 8u);
                const uint32_t p0 = __ballot_sync(FULL, (gi & 1u) != 0u), p1 = __ballot_sync(FULL, (gi & 2u) != 0u), p2 = __ballot_sync(FULL, (gi & 4u) != 0u);
                const uint32_t x = __ballot_sync(FULL, keep && (r & 0x200u));
                const uint32_t same = v & site_m & ((gi & 1u) ? p0 : ~p0) & ((gi & 2u) ? p1 : ~p1) & ((gi & 4u) ? p2 : ~p2); // this call's (site, group)
                const uint32_t slot = s * 8u + (gi & 7u);
                const uint32_t prev = gi < 8u ? s_ab[warp].gcnt[slot] : 0u;
                __syncwarp();
                if (gi < 8u)
                {
                    const uint32_t rank = (prev & 127u) + __popc(same & lt_mask);
                    w_val0[at] = __uint_as_float(rank);
                    if ((same >> lane) == 1u) // the (site, group)'s last member in this chunk carries the count on
                        s_ab[warp].gcnt[slot] = static_cast<uint8_t>((rank + 1u) | (prev & 0x80u) | ((same & x) ? 0x80u : 0u));
                }
                __syncwarp();
            }
            // val0 of a call outside every group (q < 3, or no dependent model)
            if (keep && gi >= 8u) w_val0[at] = T.val0_plain[c & 63u];
        }
        const uint32_t nonref_mask = __ballot_sync(FULL, my_nonref) & 0xfffu;
        if (lane < K2_B12) s_n[warp][lane] = static_cast<uint16_t>(my_cnt);
        if (is_dep)
        {
            __syncwarp();
            // the group starts of site `lane` (exclusive sums over its 8 groups) and the list of non-empty (site, group) pairs, site-major
            uint32_t n_ne = 0, w0 = 0, w1 = 0; // w0, w1: the site's 8 count bytes
            if (lane < K2_B12)
            {
                w0 = s_ab[warp].gcnt4[2 * lane];
                w1 = s_ab[warp].gcnt4[2 * lane + 1];
                uint32_t start = 0;
#pragma unroll
                for (uint32_t g = 0; g < 8; ++g)
                {
                    const uint32_t e = ((g < 4 ? w0 : w1) >> (8 * (g & 3u))) & 0xffu;
                    s_gstart[warp][lane][g] = static_cast<uint16_t>(start);
                    start += e & 127u;
                    if (e & 127u) ++n_ne;
                }
                s_gstart[warp][lane][8] = static_cast<uint16_t>(start);
            }
            uint32_t incl = n_ne;
#pragma unroll
            for (uint32_t d = 1; d < 16; d <<= 1)
            {
                const uint32_t t = __shfl_up_sync(FULL, incl, d);
                if (lane >= d) incl += t;
            }
            n_pairs = __shfl_sync(FULL, incl, K2_B12 - 1);
            if (lane < K2_B12)
            {
                uint32_t p = incl - n_ne;
#pragma unroll
                for (uint32_t g = 0; g < 8; ++g)
                {
                    const uint32_t e = ((g < 4 ? w0 : w1) >> (8 * (g & 3u))) & 0xffu;
                    if (e & 127u) s_pair[warp][p++] = static_cast<uint8_t>(lane * 8u + g + (e & 0x80u));
                }
            }
            // pass 2: every grouped call to gstart + rank in its site's order, (quality, call index): K2_CAP12 + 2 < 128.  Over the compacted calls,
            // whose block offsets are the exclusive sums of the sites' counts.
            uint32_t my_coff = lane < K2_B12 ? my_cnt : 0u;
#pragma unroll
            for (uint32_t d = 1; d < 16; d <<= 1)
            {
                const uint32_t t = __shfl_up_sync(FULL, my_coff, d);
                if (lane >= d) my_coff += t;
            }
            my_coff -= lane < K2_B12 ? my_cnt : 0u;
            const uint32_t n_kept = __shfl_sync(FULL, my_coff, K2_B12);
            __syncwarp();
            for (uint32_t b = 0; b < n_kept; b += 32)
            {
                const uint32_t s = k2_site_of(my_coff, b, lane);
                const uint32_t k = b + lane - __shfl_sync(FULL, my_coff, s);
                if (b + lane < n_kept)
                {
                    const uint32_t r = w_calls0[s * cap + k];
                    const uint32_t gi = k2_group(r);
                    if (gi < 8u) w_ord0[s * cap + s_gstart[warp][s][gi] + __float_as_uint(w_val0[s * cap + k])] = static_cast<uint16_t>((((r >> 3) & 63u) << 7) | k);
                }
            }
        }
        __syncwarp();
        // ---- phase B: one non-empty (site, group) pair per lane -- adjust_icalls_eprob (adjust_joint_eprob.cpp:100-180), then
        //      val0 = logf(de) + ln(1/3) (position_snp_call_pprob_digt.cpp:352) of the group's members.  A group without a neighbour-mismatch
        //      call has mismatch_frac 0, hence the tabulated exponents: no weight sums, and table reads instead of powf and logf.  Where the
        //      exponents reach the clamp within SX_K2_CLEAN_RANKS ranks only those first ranks of the sorted order are needed (below).
        if (is_dep)
        {
            for (uint32_t p = lane; p < n_pairs; p += 32)
            {
                const uint32_t pr = s_pair[warp][p], s = (pr >> 3) & 15u, g = pr & 7u;
                const bool dirty = (pr & 0x80u) != 0u;
                const uint16_t* w_calls = s_calls_all + (warp * K2_B12 + s) * cap;
                float* w_val = s_val_all + (warp * K2_B12 + s) * cap;
                const uint32_t g0 = s_gstart[warp][s][g], sz = s_gstart[warp][s][g + 1] - g0;
                uint16_t* ic = w_ord0 + s * cap + g0;
                const PKey key{};
                // the exponent chain: a clean group (mismatch_frac 0) has the tabulated one, a group with a mismatch call takes its vexp_frac
                // from the weight sums; either way only the ranks before the clamp have their own de, every later member gets depmin[q]
                bool partial = clean_ok && !dirty;
                uint32_t ranks = clean_ranks;
                float step = 0.f;
                if (!partial)
                {
                    float num = 0.f, den = 0.f; // :112-127, in pileup order (before the sort)
                    for (uint32_t k = 0; k < sz; ++k)
                    {
                        const uint32_t e = ic[k];
                        const float weight = T.weight[e >> 7];
                        den = f_add(den, weight);
                        if (w_calls[e & 127u] & 0x200u) num = f_add(num, weight);
                    }
                    float mismatch_frac = 0.f;
                    if (static_cast<double>(den) > 0.) mismatch_frac = f_div(num, den);
                    step = f_sub(1.0f, vexp_frac_of(mismatch_frac, ssd_no, ssd_one));
                    if (is_limit_vexp)
                    {
                        float vexp = 1.0f;
                        bool clamped = false;
                        ranks = 0;
                        for (int j = 0; j < SX_K2_CLEAN_RANKS && !clamped; ++j)
                        {
                            ++ranks;
                            const float next_vexp = f_mul(vexp, step);
                            clamped = (next_vexp <= min_vexp);
                            vexp = (min_vexp < next_vexp) ? next_vexp : min_vexp;
                        }
                        partial = clamped;
                    }
                }
                if (partial)
                {
                    // std::sort ends in an insertion sort, which is stable, so its order is the stable descending sort of what the partitioning
                    // leaves (for <= 16 members: of the pileup order).  One pass keeps the first SX_K2_CLEAN_RANKS of that order in registers (ties
                    // in scan order) and gives every member val0_min[q]; the first `ranks` are then overwritten.  The group is not sorted.
                    if (sz > 16) sx_introsort_loop_desc<K2_SORT_STACK12>(ic, static_cast<int>(sz), key);
                    uint32_t top[SX_K2_CLEAN_RANKS]; // packed (q << 7 | call index), quality-descending; 0 = empty (a member has q >= 3)
#pragma unroll
                    for (int j = 0; j < SX_K2_CLEAN_RANKS; ++j) top[j] = 0u;
                    for (uint32_t k = 0; k < sz; ++k)
                    {
                        const uint32_t e = ic[k], q = e >> 7;
                        w_val[e & 127u] = T.val0_min[q];
#pragma unroll
                        for (int j = SX_K2_CLEAN_RANKS - 1; j > 0; --j)
                        {
                            if ((top[j - 1] >> 7) < q) top[j] = top[j - 1];
                            else if ((top[j] >> 7) < q) top[j] = e;
                        }
                        if ((top[0] >> 7) < q) top[0] = e;
                    }
#pragma unroll
                    for (uint32_t j = 0; j < SX_K2_CLEAN_RANKS; ++j)
                        if (j < sz) ic[j] = static_cast<uint16_t>(top[j]); // the group's order is not needed any more
                    const uint32_t nr = min(ranks, sz);
                    if (clean_ok && !dirty)
                    {
                        for (uint32_t j = 0; j < nr; ++j) w_val[ic[j] & 127u] = T.val0_clean[j][ic[j] >> 7];
                    }
                    else
                    {
                        float vexp = 1.0f;
                        for (uint32_t j = 0; j < nr; ++j)
                        {
                            const uint32_t q = ic[j] >> 7;
                            w_val[ic[j] & 127u] = f_add(sx_logf(dependent_eprob(T.eprob[q], vexp)), log_one_third);
                            const float next_vexp = f_mul(vexp, step);
                            vexp = (min_vexp < next_vexp) ? next_vexp : min_vexp; // std::max(min_vexp, next_vexp)
                        }
                    }
                    continue;
                }
                // no clamp within SX_K2_CLEAN_RANKS ranks (or none at all): the whole order
                sx_stdsort_desc<K2_SORT_STACK12>(ic, sz, key);
                float vexp = 1.0f;
                bool is_min_vexp = false;
                for (uint32_t k = 0; k < sz; ++k)
                {
                    const uint32_t idx = ic[k] & 127u, q = ic[k] >> 7;
                    if (!is_min_vexp)
                    {
                        w_val[idx] = f_add(sx_logf(dependent_eprob(T.eprob[q], vexp)), log_one_third);
                        const float next_vexp = f_mul(vexp, step);
                        if (is_limit_vexp)
                        {
                            is_min_vexp = (next_vexp <= min_vexp);
                            vexp = (min_vexp < next_vexp) ? next_vexp : min_vexp; // std::max(min_vexp, next_vexp)
                        }
                        else
                        {
                            vexp = next_vexp;
                        }
                    }
                    else
                    {
                        w_val[idx] = T.val0_min[q]; // dependent_prob_cache: get_dependent_eprob(q, min_vexp)
                    }
                }
            }
        }
        __syncwarp();
        // ---- phase C, three sites at a time: likelihoods and PLs
        uint32_t computed_mask = 0;
        for (uint32_t s0 = 0; s0 < nb; s0 += 3)
        {
            const uint32_t s = s0 + sub;
            const bool have = s < nb;
            const uint32_t site = have ? base + s : base;
            const uint16_t* w_calls = s_calls_all + (warp * K2_B12 + (have ? s : 0)) * cap;
            const float* w_val = s_val_all + (warp * K2_B12 + (have ? s : 0)) * cap;
            const uint32_t n = have ? s_n[warp][s] : 0u;
            const uint32_t info = __shfl_sync(FULL, my_info, have ? s : 0u);
            const uint32_t ref_gt = info & 7u;
            const bool nonref = (nonref_mask >> (have ? s : 0)) & 1u;
            const bool computed = have && (ref_gt < 4u) && (is_always_test || nonref);
            sx_digt_result* res = out + site;
            if (have && !computed && sl < 10)
            {
                uint32_t* w = reinterpret_cast<uint32_t*>(res);
                for (uint32_t i = sl; i < sizeof(sx_digt_result) / 4; i += 10) w[i] = 0u;
            }
            __syncwarp();
            if (have && !computed && sl == 0)
            {
                res->ref_gt = (ref_gt < 4u) ? ref_gt : 0u;
                res->n_used_calls = n;
            }
            const bool act = computed && sl < 10;
            const uint32_t n_act = computed ? n : 0u;
            const uint32_t n_loop = max(max(__shfl_sync(FULL, n_act, 0), __shfl_sync(FULL, n_act, 10)), __shfl_sync(FULL, n_act, 20));
            // branch-free: every lane loads every step (addresses stay inside the warp's arrays) and the lanes past their site's end add +0.0f,
            // which leaves a sum that started at +0.0f unchanged bit for bit
            const uint32_t e2s = expect2_pack(sl < 10u ? sl : 0u) << 2; // expect2 << 2: the table offset of {val1, val2} in bytes
            const uint32_t a_tab = smem_u32(s_val12) - 4u;
            const uint32_t n_mine = act ? n : 0u;
            uint32_t a_c = smem_u32(w_calls), a_v = smem_u32(w_val);
            float lh = 0.f;
#pragma unroll 4
            for (uint32_t i = 0; i < n_loop; ++i, a_c += 2u, a_v += 4u)
            {
                const uint32_t r = lds_u16(a_c);
                const uint32_t k4 = (e2s >> (r >> 13)) & 12u;
                const float v = lds_f32(k4 ? a_tab + (r & 0x1f8u) + k4 : a_v);
                lh = f_add(lh, i < n_mine ? v : 0.f);
            }
            const bool haploid = have && (info & 8u);
            const uint32_t gtcount = haploid ? 4u : 10u;
            float lmax = __shfl_sync(FULL, lh, sbase);
            for (uint32_t g = 1; g < 10; ++g)
            {
                const float v = __shfl_sync(FULL, lh, sbase + g);
                if (g < gtcount && v > lmax) lmax = v;
            }
            uint32_t pl = 0;
            if (act && sl < gtcount) pl = static_cast<uint32_t>(ln_error_prob_to_qphred_f(f_sub(lh, lmax), ln10f));
            if (act)
            {
                res->lhood[sl] = lh;
                res->phredLoghood[sl] = pl;
                s_ab[warp].lh[s][sl] = lh; // the row phase D reads
            }
            const uint32_t cm = __ballot_sync(FULL, computed && sl == 0u); // lanes 0, 10, 20
            computed_mask |= ((cm & 1u) | ((cm >> 9) & 2u) | ((cm >> 18) & 4u)) << s0;
        }
        __syncwarp();
        // ---- phase D: the posteriors, one (site, prior) pair per lane -- lanes 0-11 the genomic prior of sites 0-11, lanes 12-23 the polymorphic one.
        //      calculate_result_set is a 10-term reduction with a double exp per term and two double log10: on 10 lanes per site and prior it
        //      was issued 8 times per batch for the whole warp; serially per lane it is
        //      issued once.  Same operations in the same order per (site, prior), so the same bits.
        {
            const uint32_t ps = lane < 12u ? lane : lane - 12u;
            const bool pact = lane < 24u && ps < nb && ((computed_mask >> ps) & 1u);
            const uint32_t site = base + (pact ? ps : 0u);
            const uint32_t info = __shfl_sync(FULL, my_info, pact ? ps : 0u);
            const uint32_t ref_gt = info & 3u; // < 4 where it is used (pact)
            sx_digt_result* res = out + site;
            rs_out r;
            r.ref_pprob = 0.0;
            r.max_gt = 0;
            r.snp_qphred = 0;
            r.max_gt_qphred = 0;
            if (pact)
            {
                const bool haploid = (info & 8u) != 0u;
                const float* pri = T.lnprior[haploid ? 1 : 0][ref_gt][0] + (lane < 12u ? 0 : 10);
                const float* lh10 = s_ab[warp].lh[ps];
                double e[10];
                double mx = 0.0;
#pragma unroll
                for (int gt = 0; gt < 10; ++gt)
                {
                    e[gt] = static_cast<double>(f_add(lh10[gt], pri[gt]));
                    if (gt == 0 || e[gt] > mx)
                    {
                        mx = e[gt];
                        r.max_gt = gt;
                    }
                }
                double sum = 0.0;
#pragma unroll
                for (int gt = 0; gt < 10; ++gt)
                {
                    e[gt] = sx_exp(d_sub(e[gt], mx));
                    sum = d_add(sum, e[gt]);
                }
                sum = d_div(1.0, sum);
                double comp = 0.0;
#pragma unroll
                for (int gt = 0; gt < 10; ++gt)
                {
                    const double pg = d_mul(e[gt], sum);
                    if (gt != (int)r.max_gt) comp = d_add(comp, pg);
                    if (gt == (int)ref_gt) r.ref_pprob = pg;
                }
                r.snp_qphred = error_prob_to_qphred_d(r.ref_pprob);
                r.max_gt_qphred = error_prob_to_qphred_d(comp);
                sx_digt_result_set* dst = lane < 12u ? &res->genome : &res->poly;
                dst->ref_pprob = r.ref_pprob;
                dst->max_gt = r.max_gt;
                dst->snp_qphred = r.snp_qphred;
                dst->max_gt_qphred = r.max_gt_qphred;
                dst->pad = 0;
            }
            // strand bias, SNP sites only (rare): the fwd-specific and rev-specific sums of the called genotype (:522-533) on lanes 0 and 1
            double strand_bias = 0.0;
            uint32_t snp_mask = __ballot_sync(FULL, pact && lane < 12u && r.snp_qphred != 0);
            while (snp_mask)
            {
                const uint32_t s = __ffs(snp_mask) - 1u;
                snp_mask &= snp_mask - 1u;
                const uint32_t tgt = __shfl_sync(FULL, r.max_gt, s);
                const uint16_t* w_calls = s_calls_all + (warp * K2_B12 + s) * cap;
                const float* w_val = s_val_all + (warp * K2_B12 + s) * cap;
                const uint32_t ref_s = __shfl_sync(FULL, my_info, s) & 3u;
                float ls = 0.f;
                if (lane < 2u)
                {
                    const uint32_t e2_t = expect2_pack(tgt), e2_ref = expect2_pack(ref_s);
                    const uint32_t n = s_n[warp][s];
                    for (uint32_t i = 0; i < n; ++i)
                    {
                        const uint32_t c = w_calls[i]; // repacked: obs << 14 | q << 3 | fwd
                        const uint32_t q = (c >> 3) & 63u, obs = c >> 14, fwd = c & 1u;
                        const bool force_ref = ((lane == 0u) != (fwd != 0u)); // lane 0: the fwd-specific sum (reverse-strand calls forced to the reference), 1: rev-specific
                        const uint32_t k = ((force_ref ? e2_ref : e2_t) >> (2u * obs)) & 3u;
                        ls = f_add(ls, (k == 0u) ? w_val[i] : s_val12[2u * q + k - 1u]);
                    }
                }
                const float lf = __shfl_sync(FULL, ls, 0), lr = __shfl_sync(FULL, ls, 1), l0 = s_ab[warp].lh[s][tgt];
                if (lane == s) strand_bias = static_cast<double>(f_sub((lf < lr) ? lr : lf, l0));
            }
            if (pact && lane < 12u)
            {
                res->strand_bias = strand_bias;
                res->ref_gt = ref_gt;
                res->is_computed = 1;
                res->n_used_calls = s_n[warp][ps];
                res->pad = 0;
            }
        }
        __syncwarp();
    }
}

// out[0]: the deepest site; out[1]: the most raw calls of one twelve-site batch (the twelve-site kernel's batches start at multiples of K2_B12)
__global__ void k2_max_site_kernel(const uint32_t* __restrict__ site_off, uint32_t n_sites, uint32_t* __restrict__ out)
{
    uint32_t m = 0, mb = 0;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_sites; i += gridDim.x * blockDim.x)
    {
        const uint32_t o = site_off[i];
        m = max(m, site_off[i + 1] - o);
        if (i % K2_B12 == 0) mb = max(mb, site_off[min(i + K2_B12, n_sites)] - o);
    }
    for (int d = 16; d; d >>= 1)
    {
        m = max(m, __shfl_xor_sync(FULL, m, d));
        mb = max(mb, __shfl_xor_sync(FULL, mb, d));
    }
    if ((threadIdx.x & 31) == 0 && m) atomicMax(out, m);
    if ((threadIdx.x & 31) == 0 && mb) atomicMax(out + 1, mb);
}

// the same two numbers for a host batch
void max_block_host(const sx_pileup_batch* b, uint32_t* max_block)
{
    uint32_t mb = 0;
    for (uint32_t s = 0; s < b->n_sites; s += K2_B12) mb = std::max(mb, b->site_off[std::min<uint32_t>(s + K2_B12, b->n_sites)] - b->site_off[s]);
    *max_block = mb;
}

// max_block: the most raw calls of one twelve-site batch (read only when the twelve-site kernel runs)
int germline_run(sx_ctx* ctx, const sx_pileup_batch* d, int is_always_test, sx_digt_result* out_dev, uint32_t* de_off_dev, float* de_dev, uint32_t max_site,
                 uint32_t max_block)
{
    if (max_site > K2_CAP_BIG)
        return sx_fail(ctx, SX_ERR_UNSUPPORTED, "sx_site_gl_germline: a site holds %u calls; the kernel handles at most %d per site", max_site, K2_CAP_BIG);
    if (de_dev == nullptr && max_site <= K2_CAP12)
    {
        // twelve sites per warp: 8 bytes of shared memory per call slot
        const uint32_t per_cta = K2_WARPS * K2_B12;
        // per-site stride: even, and never a multiple of 16 slots -- phase C reads slot i of three consecutive sites in one instruction, and
        // a stride of 32 (64) slots put the three float (16-bit) words on one bank (most shared-memory wavefronts were then bank conflicts)
        uint32_t cap = std::max<uint32_t>(18, (max_site + 1) & ~1u);
        if (cap % 16 == 0) cap += 2;
        // the order region also takes a batch's raw block with up to 7 calls before it and 7 after (whole 16-byte words): 12 * cap slots
        // suffice unless nearly every site of a batch is the deepest; a multiple of 8 slots keeps every warp's region 16-byte aligned
        const uint32_t ord_stride = std::max<uint32_t>(K2_B12 * cap, (max_block + 14 + 7) & ~7u);
        const size_t smem = (size_t)K2_WARPS * (K2_B12 * cap * 6 + ord_stride * 2);
        int occ = 4;
        SX_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k2a_germline12_kernel, K2_WARPS * 32, smem));
        const int grid12 = static_cast<int>(std::min<uint32_t>((d->n_sites + per_cta - 1) / per_cta, (uint32_t)(ctx->sm_count * std::max(1, occ))));
        k2a_germline12_kernel<<<grid12, K2_WARPS * 32, smem, ctx->s_compute>>>(d->site_off, d->calls, d->ref_base, d->ploidy, d->n_sites, is_always_test, ctx->d_tables, out_dev,
                                                                             ctx->d_status, cap, ord_stride);
        SX_CUDA(ctx, cudaGetLastError());
        return SX_OK;
    }
    if (max_site <= K2_CAP_SMEM)
    {
        // every site fits the shared-memory cap: four sites per warp, 8 bytes of shared memory per call slot
        const uint32_t per_cta = K2_WARPS * K2_BATCH;
        const uint32_t cap = std::max<uint32_t>(32, (max_site + 31) & ~31u);
        const size_t smem = (size_t)per_cta * cap * 8;
        int occ = 6;
        SX_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k2a_germline_batch_kernel<K2_BATCH>, K2_WARPS * 32, smem));
        const int grid4 = static_cast<int>(std::min<uint32_t>((d->n_sites + per_cta - 1) / per_cta, (uint32_t)(ctx->sm_count * std::max(1, occ))));
        k2a_germline_batch_kernel<K2_BATCH><<<grid4, K2_WARPS * 32, smem, ctx->s_compute>>>(d->site_off, d->calls, d->ref_base, d->ploidy, d->n_sites, is_always_test,
                                                                                          ctx->d_tables, out_dev, de_off_dev, de_dev, ctx->d_status, cap, nullptr);
        SX_CUDA(ctx, cudaGetLastError());
        return SX_OK;
    }
    // a deeper site: one site per warp, K2_CAP_SMEM calls in shared memory, a deeper site in the warp's K2_CAP_BIG-call region of the scratch
    const int grid = static_cast<int>(std::min<uint32_t>((d->n_sites + K2_WARPS - 1) / K2_WARPS, (uint32_t)ctx->sm_count * 8));
    unsigned char* scratch = nullptr;
    const int rc = sx_take(ctx, SX_SLOT_K2A_SCRATCH, (size_t)grid * K2_WARPS * K2_CAP_BIG * 8, scratch, 0);
    if (rc) return rc;
    k2a_germline_batch_kernel<1><<<grid, K2_WARPS * 32, (size_t)K2_WARPS * K2_CAP_SMEM * 8, ctx->s_compute>>>(d->site_off, d->calls, d->ref_base, d->ploidy, d->n_sites,
                                                                                                           is_always_test, ctx->d_tables, out_dev, de_off_dev, de_dev,
                                                                                                           ctx->d_status, K2_CAP_SMEM, scratch);
    SX_CUDA(ctx, cudaGetLastError());
    return SX_OK;
}

// out[0]: the deepest site, out[1]: the largest twelve-site batch, in one round trip
int max_site_dev(sx_ctx* ctx, const uint32_t* site_off_dev, uint32_t n_sites, uint32_t* out)
{
    uint32_t* d = nullptr;
    int rc = sx_take(ctx, SX_SLOT_K2A_MAX_SITE, 2, d, 0);
    if (rc) return rc;
    SX_CUDA(ctx, cudaMemsetAsync(d, 0, 2 * sizeof(uint32_t), ctx->s_compute));
    k2_max_site_kernel<<<std::min<uint32_t>((n_sites + 255) / 256, 1184), 256, 0, ctx->s_compute>>>(site_off_dev, n_sites, d);
    SX_CUDA(ctx, cudaMemcpyAsync(out, d, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->s_compute));
    SX_CUDA(ctx, cudaStreamSynchronize(ctx->s_compute));
    return SX_OK;
}
} // namespace

cudaError_t sx_k2a_init_tables(sx_tables* d_tables)
{
    k2a_init_tables_kernel<<<1, 96>>>(d_tables);
    const cudaError_t e = cudaGetLastError();
    return e != cudaSuccess ? e : cudaDeviceSynchronize();
}

extern "C" int sx_site_gl_germline_dev(sx_ctx* ctx, const sx_pileup_batch* d, int is_always_test, sx_digt_result* out_dev)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    if (!d || !out_dev || !d->site_off || !d->calls || !d->ref_base) return sx_fail(ctx, SX_ERR_ARG, "sx_site_gl_germline_dev: NULL argument");
    if (d->n_sites == 0) return SX_OK;
    const int rc = sx_run_timed(ctx, [&](unsigned* launches) { return sx_k2a_run(ctx, d, is_always_test, out_dev, launches); });
    if (rc) return rc;
    return sx_check_status(ctx, "sx_site_gl_germline");
}

// upload a host pileup batch into host slots host_base..host_base+5; returns the device view
int sx_upload_pileup(sx_ctx* ctx, const sx_pileup_batch* b, int host_base, sx_pileup_batch* d, uint32_t* max_site)
{
    if (!b->site_off || !b->calls || !b->ref_base) return sx_fail(ctx, SX_ERR_ARG, "pileup batch: NULL array");
    *d = *b;
    int rc;
    const size_t n(b->n_sites);
    uint32_t m = 0;
    for (uint32_t s = 0; s < b->n_sites; ++s)
    {
        if (b->site_off[s + 1] < b->site_off[s]) return sx_fail(ctx, SX_ERR_ARG, "pileup batch: site_off not monotone at site %u", s);
        m = std::max(m, b->site_off[s + 1] - b->site_off[s]);
    }
    *max_site = m;
    if ((rc = sx_upload(ctx, sx_host_slot(host_base), b->site_off, n + 1, d->site_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(host_base + 1), b->calls, b->site_off[b->n_sites], d->calls, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(host_base + 2), b->ref_base, n, d->ref_base, 16))) return rc;
    if (b->ploidy && (rc = sx_upload(ctx, sx_host_slot(host_base + 3), b->ploidy, n, d->ploidy, 16))) return rc;
    if (b->t2_off)
    {
        if (!b->t2_calls) return sx_fail(ctx, SX_ERR_ARG, "pileup batch: t2_off without t2_calls");
        if ((rc = sx_upload(ctx, sx_host_slot(host_base + 4), b->t2_off, n + 1, d->t2_off, 16))) return rc;
        if ((rc = sx_upload(ctx, sx_host_slot(host_base + 5), b->t2_calls, b->t2_off[b->n_sites], d->t2_calls, 16))) return rc;
        uint32_t m2 = 0;
        for (uint32_t s = 0; s < b->n_sites; ++s) m2 = std::max(m2, b->site_off[s + 1] - b->site_off[s] + b->t2_off[s + 1] - b->t2_off[s]);
        *max_site = std::max(*max_site, m2);
    }
    return SX_OK;
}

extern "C" int sx_site_gl_germline(sx_ctx* ctx, const sx_pileup_batch* b, int is_always_test, sx_digt_result* out_host)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    if (!b || !out_host) return sx_fail(ctx, SX_ERR_ARG, "sx_site_gl_germline: NULL argument");
    if (b->n_sites == 0) return SX_OK;
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    sx_pileup_batch d;
    uint32_t max_site = 0;
    sx_call_timer t(ctx);
    int rc = sx_upload_pileup(ctx, b, 9, &d, &max_site);
    if (rc) return rc;
    sx_digt_result* d_out = nullptr;
    if ((rc = sx_take(ctx, sx_host_slot(15), b->n_sites, d_out, 0))) return rc;
    uint32_t max_block = 0;
    max_block_host(b, &max_block);
    if ((rc = germline_run(ctx, &d, is_always_test, d_out, nullptr, nullptr, max_site, max_block))) return rc;
    if ((rc = sx_download(ctx, out_host, d_out, b->n_sites))) return rc;
    if ((rc = t.finish(1))) return rc; // (the deepest site was found on the host)
    return sx_check_status(ctx, "sx_site_gl_germline");
}

extern "C" int sx_dependent_eprob(sx_ctx* ctx, const sx_pileup_batch* b, uint32_t* out_off_host, float* de_host)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    if (!b || !out_off_host || !de_host) return sx_fail(ctx, SX_ERR_ARG, "sx_dependent_eprob: NULL argument");
    if (b->n_sites == 0)
    {
        out_off_host[0] = 0;
        return SX_OK;
    }
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    // offsets of the cleaned calls (host side: the filter bit is in the input)
    uint32_t off = 0;
    for (uint32_t s = 0; s < b->n_sites; ++s)
    {
        out_off_host[s] = off;
        for (uint32_t i = b->site_off[s]; i < b->site_off[s + 1]; ++i) off += !((b->calls[i] >> 12) & 1u);
    }
    out_off_host[b->n_sites] = off;
    sx_pileup_batch d;
    uint32_t max_site = 0;
    int rc = sx_upload_pileup(ctx, b, 9, &d, &max_site);
    if (rc) return rc;
    uint32_t* d_off = nullptr;
    float* d_de = nullptr;
    if ((rc = sx_upload(ctx, sx_host_slot(16), out_off_host, (size_t)b->n_sites + 1, d_off, 0))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(17), off, d_de, 16))) return rc;
    if ((rc = germline_run(ctx, &d, 1, nullptr, d_off, d_de, max_site, 0))) return rc;
    if ((rc = sx_download(ctx, de_host, d_de, off))) return rc;
    SX_CUDA(ctx, cudaStreamSynchronize(ctx->s_compute));
    ctx->timing.launches = 1;
    ctx->total_launches += 1;
    return sx_check_status(ctx, "sx_dependent_eprob");
}

// K2a's launcher: one 8-byte round trip (the deepest column, the largest twelve-site block) picks and sizes the kernel
int sx_k2a_run(sx_ctx* ctx, const sx_pileup_batch* d, int is_always_test, sx_digt_result* out_dev, unsigned* launches)
{
    if (d->n_sites == 0) return SX_OK;
    uint32_t max_site[2] = {0, 0};
    int rc = max_site_dev(ctx, d->site_off, d->n_sites, max_site);
    if (rc) return rc;
    rc = germline_run(ctx, d, is_always_test, out_dev, nullptr, nullptr, max_site[0], max_site[1]);
    *launches += 2;
    return rc;
}
