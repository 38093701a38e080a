// k3_global_align.cu -- K3 global_align: affine-gap global alignment of a haplotype to a reference segment, with traceback.
//
// Replaces GlobalAligner<int>::align   (/root/reference/src/c++/lib/alignment/GlobalAlignerImpl.hh:36-228),
//          backTraceAlignment          (alignment/SingleRefAlignerSharedImpl.hh:80-170) and
//          apath_add_seqmatch          (blt_util/align_path_impl.hh:36-86)
// as called from ActiveRegionProcessor::discoverIndelsAndMismatches (starling_common/ActiveRegionProcessor.cpp:591).
//
// This file holds the entry points and the kernel for LARGE matrices (Q > 128 or R > 255, and batches whose penalties do not fit
// the key encoding of k3_group.cu, which takes everything else first -- see sx_k3_group_launch).
//
// One warp per DP matrix.  Lane l owns the strip of T = ceil(Q/32) consecutive query rows and keeps the three state scores
// of its rows IN REGISTERS (T is a template parameter up to 4, i.e. Q <= 128; longer queries fall back to a shared-memory
// strip).  The warp sweeps the matrix as an anti-diagonal wavefront: lane l is at reference column t-l at step t, and the
// scores of the row above / the diagonal cross strips through three __shfl_up per step.  The 3 x 2-bit back pointers of every
// cell go to a (Q+1) x (R+1) byte matrix in shared memory, so HBM sees only the Q+R input bytes and the result.
// The traceback is a pointer chase (one lane); the '='/'X' expansion and run-length encoding of the path is done by the whole
// warp with ballot/popc scans.  Scores are int32 and max3 keeps the reference's first-argument-wins tie rule
// (alignment/AlignerBase.hh:71-92), so score, beginPos and CIGAR are bit-exact.
#include "k3_common.cuh"
#include "sx_internal.h"

#include <algorithm>

namespace
{
using namespace k3;
constexpr int K3_WARPS = 4;

struct problem_smem
{
    uint8_t* ptr;
    int *sM, *sD, *sI;
    char *qs, *rs;
    uint8_t* steps;
};

__device__ __forceinline__ problem_smem carve(unsigned char* base, uint32_t Q, uint32_t R)
{
    const k3_slot_layout L = k3_slot(Q, R);
    const uint32_t T = (Q + 31) / 32;
    problem_smem p;
    p.ptr = base;
    p.sM = reinterpret_cast<int*>(base + L.strips);
    p.sD = p.sM + 32 * T;
    p.sI = p.sD + 32 * T;
    p.qs = reinterpret_cast<char*>(base + L.query);
    p.rs = reinterpret_cast<char*>(base + L.ref);
    p.steps = base + L.steps;
    return p;
}

// The wavefront with T rows per lane in registers (Q <= 128), written branch-free inside a step: every lane runs all T rows; rows past
// the query end (only in the last active lane) compute discarded values and skip the pointer store by predicate; DP row 0 (lane 0's
// "row above") is a select between closed forms instead of a divergent branch.  Leaves the final-column scores in S.sM/sD/sI.
template <int T>
__device__ __forceinline__ void dp_register_strip(const sx_ga_scores& sc, const problem_smem& S, uint32_t Q, uint32_t R, uint32_t lane, bt_state& colbt)
{
    const uint32_t W = R + 1;
    const uint32_t last_lane = (Q - 1) / T;
    const uint32_t row0 = lane * T; // query index of this lane's first row
    int rM[T], rD[T], rI[T];
    char qc[T];
    uint32_t prow[T];
#pragma unroll
    for (int r = 0; r < T; ++r)
    {
        const uint32_t qi = row0 + r;
        col0_scores(sc, (int)qi + 1, rM[r], rD[r], rI[r]);
        qc[r] = qi < Q ? S.qs[qi] : 0;
        prow[r] = (qi + 1) * W + 1;
    }
    int sendM = 0, sendD = 0, sendI = 0;
    int prevRecvM = 0, prevRecvD = 0, prevRecvI = 0;
    const uint32_t n_steps = R + last_lane;
    const int s_match = sc.match, s_mismatch = sc.mismatch, s_open = sc.open, s_extend = sc.extend, s_insdel = sc.insertDelete;
    const int row0M = sc.isRequireEdgeDeletion ? BAD : 0;
    const bool req_del = sc.isRequireEdgeDeletion != 0;
    int c0M, c0D, c0I; // initial column at the DP row above this strip (the diagonal for j == 0)
    col0_scores(sc, (int)row0, c0M, c0D, c0I);
    const uint32_t r_last = (Q - 1) - last_lane * T; // strip-relative index of DP row Q in the last lane
    const bool is_lane0 = lane == 0;
    for (uint32_t t = 0; t < n_steps; ++t)
    {
        const int recvM = __shfl_up_sync(FULL, sendM, 1);
        const int recvD = __shfl_up_sync(FULL, sendD, 1);
        const int recvI = __shfl_up_sync(FULL, sendI, 1);
        const int j = static_cast<int>(t) - static_cast<int>(lane);
        if (j >= 0 && j < static_cast<int>(R) && lane <= last_lane)
        {
            const char rc = S.rs[j];
            const bool j0 = j == 0;
            // row above in this column: DP row 0 at matrix column j+1 for lane 0, else what the previous lane sent last step
            int upM = is_lane0 ? row0M : recvM;
            int upD = is_lane0 ? (req_del ? s_open + (j + 1) * s_extend : BAD) : recvD;
            int upI = is_lane0 ? BAD : recvI;
            // diagonal: initial column for j == 0; else DP row 0 at matrix column j (lane 0) / what arrived one step earlier
            int dgM = j0 ? c0M : (is_lane0 ? row0M : prevRecvM);
            int dgD = j0 ? c0D : (is_lane0 ? (req_del ? s_open + j * s_extend : BAD) : prevRecvD);
            int dgI = j0 ? c0I : (is_lane0 ? BAD : prevRecvI);
            int mQ = 0;
#pragma unroll
            for (int r = 0; r < T; ++r)
            {
                const int lfM = rM[r], lfD = rD[r], lfI = rI[r];
                int m, d, ins;
                const uint32_t pm = max3(m, dgM, dgD, dgI);
                m += (qc[r] == rc) ? s_match : s_mismatch;
                const uint32_t pd = max3(d, lfM + s_open, lfD, lfI + s_insdel);
                d = j0 ? BAD : d + s_extend;
                const uint32_t pi = max3(ins, upM + s_open, BAD, upI);
                ins += s_extend;
                if (r == 0) ins = (row0 == 0) ? BAD : ins; // queryIndex 0
                if (row0 + r < Q) S.ptr[prow[r] + j] = static_cast<uint8_t>(pm | (pd << 2) | (pi << 4));
                dgM = lfM;
                dgD = lfD;
                dgI = lfI;
                upM = m;
                upD = d;
                upI = ins;
                rM[r] = m;
                rD[r] = d;
                rI[r] = ins;
                if ((uint32_t)r == r_last) mQ = m;
            }
            sendM = upM;
            sendD = upD;
            sendI = upI;
            if (lane == last_lane && !req_del) update_bt(colbt, mQ, j + 1, Q, ST_MATCH); // :170-175
        }
        prevRecvM = recvM;
        prevRecvD = recvD;
        prevRecvI = recvI;
    }
#pragma unroll
    for (int r = 0; r < T; ++r)
    {
        S.sM[r * 32 + lane] = rM[r];
        S.sD[r * 32 + lane] = rD[r];
        S.sI[r * 32 + lane] = rI[r];
    }
    __syncwarp();
}

// The wavefront with T = ceil(Q/32) > 4 rows per lane (Q > 128): the strip lives in shared memory, at S.sM/sD/sI[r * 32 + lane].
__device__ __forceinline__ void dp_shared_strip(const sx_ga_scores& sc, const problem_smem& S, uint32_t Q, uint32_t R, uint32_t lane, bt_state& colbt)
{
    const uint32_t T = (Q + 31) / 32;
    const uint32_t W = R + 1;
    const uint32_t last_lane = (Q - 1) / T;
    const uint32_t row0 = lane * T; // query index of this lane's first row
    for (uint32_t r = 0; r < T; ++r)
    {
        int m, d, i;
        col0_scores(sc, (int)(row0 + r) + 1, m, d, i);
        S.sM[r * 32 + lane] = m;
        S.sD[r * 32 + lane] = d;
        S.sI[r * 32 + lane] = i;
    }
    int sendM = 0, sendD = 0, sendI = 0;
    int prevRecvM = 0, prevRecvD = 0, prevRecvI = 0;
    const uint32_t n_steps = R + last_lane;
    for (uint32_t t = 0; t < n_steps; ++t)
    {
        const int recvM = __shfl_up_sync(FULL, sendM, 1);
        const int recvD = __shfl_up_sync(FULL, sendD, 1);
        const int recvI = __shfl_up_sync(FULL, sendI, 1);
        const int j = static_cast<int>(t) - static_cast<int>(lane);
        if (j >= 0 && j < static_cast<int>(R) && lane <= last_lane)
        {
            const char rc = S.rs[j];
            int upM, upD, upI, dgM, dgD, dgI;
            if (lane == 0)
            {
                row0_scores(sc, j + 1, upM, upD, upI);
                if (j == 0) col0_scores(sc, 0, dgM, dgD, dgI);
                else row0_scores(sc, j, dgM, dgD, dgI);
            }
            else
            {
                upM = recvM;
                upD = recvD;
                upI = recvI;
                if (j == 0) col0_scores(sc, (int)row0, dgM, dgD, dgI);
                else
                {
                    dgM = prevRecvM;
                    dgD = prevRecvD;
                    dgI = prevRecvI;
                }
            }
            int m = 0, d = 0, ins = 0;
            for (uint32_t r = 0; r < T; ++r)
            {
                const uint32_t qi = row0 + r;
                if (qi >= Q) break;
                const uint32_t idx = r * 32 + lane;
                const int lfM = S.sM[idx], lfD = S.sD[idx], lfI = S.sI[idx];
                const uint32_t pm = max3(m, dgM, dgD, dgI);
                m += (S.qs[qi] == rc) ? sc.match : sc.mismatch;
                const uint32_t pd = max3(d, lfM + sc.open, lfD, lfI + sc.insertDelete);
                d += sc.extend;
                if (j == 0) d = BAD;
                const uint32_t pi = max3(ins, upM + sc.open, BAD, upI);
                ins += sc.extend;
                if (qi == 0) ins = BAD;
                S.ptr[(qi + 1) * W + (j + 1)] = static_cast<uint8_t>(pm | (pd << 2) | (pi << 4));
                dgM = lfM;
                dgD = lfD;
                dgI = lfI;
                upM = m;
                upD = d;
                upI = ins;
                S.sM[idx] = m;
                S.sD[idx] = d;
                S.sI[idx] = ins;
            }
            sendM = m;
            sendD = d;
            sendI = ins;
            if (lane == last_lane && !sc.isRequireEdgeDeletion) update_bt(colbt, m, j + 1, Q, ST_MATCH); // :170-175, m is row Q's match score
        }
        prevRecvM = recvM;
        prevRecvD = recvD;
        prevRecvI = recvI;
    }
    __syncwarp();
}

__global__ void __launch_bounds__(K3_WARPS * 32) k3_global_align_kernel(const char* __restrict__ query_pool, const char* __restrict__ ref_pool,
                                                                        const uint32_t* __restrict__ query_off, const uint32_t* __restrict__ ref_off, uint32_t n,
                                                                        uint32_t max_ops, sx_ga_scores sc, sx_ga_result* __restrict__ res,
                                                                        uint32_t* __restrict__ cigar, uint32_t slot_bytes, const uint32_t* __restrict__ order)
{
    extern __shared__ __align__(16) unsigned char smem[];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t nwarps = blockDim.x >> 5;
    unsigned char* slot = smem + (size_t)warp * slot_bytes;
    // `order`: the list of problem indices this launch owns (n entries)
    for (uint32_t k = blockIdx.x * nwarps + warp; k < n; k += gridDim.x * nwarps)
    {
        const uint32_t prob = order[k];
        const uint32_t Q = query_off[prob + 1] - query_off[prob];
        const uint32_t R = ref_off[prob + 1] - ref_off[prob];
        if (Q == 0 || R == 0 || k3_slot_bytes(Q, R) > slot_bytes)
        {
            if (lane == 0)
            {
                res[prob].score = 0;
                res[prob].beginPos = 0;
                res[prob].n_ops = 0;
                res[prob].status = 2;
            }
            continue;
        }
        const problem_smem S = carve(slot, Q, R);
        const uint32_t T = (Q + 31) / 32;
        const uint32_t W = R + 1;
        for (uint32_t i = lane; i < Q; i += 32) S.qs[i] = query_pool[query_off[prob] + i];
        for (uint32_t i = lane; i < R; i += 32) S.rs[i] = ref_pool[ref_off[prob] + i];
        // column 0 of the pointer matrix (GlobalAlignerImpl.hh:69-88) and row 0, columns 1..R (:104-126)
        {
            const uint8_t c0 = static_cast<uint8_t>(ST_MATCH | (ST_MATCH << 2) | ((sc.isAllowEdgeInsertion ? ST_INSERT : ST_MATCH) << 4));
            const uint8_t r0 = static_cast<uint8_t>(ST_MATCH | ((sc.isRequireEdgeDeletion ? ST_DELETE : ST_MATCH) << 2) | (ST_MATCH << 4));
            for (uint32_t qi = lane; qi <= Q; qi += 32) S.ptr[qi * W] = c0;
            for (uint32_t j = lane + 1; j <= R; j += 32) S.ptr[j] = r0;
        }
        __syncwarp();

        bt_state colbt{0, ST_MATCH, 0, 0, false}; // row-Q match candidates per column (only when !isRequireEdgeDeletion)
        switch (T)
        {
        case 1: dp_register_strip<1>(sc, S, Q, R, lane, colbt); break;
        case 2: dp_register_strip<2>(sc, S, Q, R, lane, colbt); break;
        case 3: dp_register_strip<3>(sc, S, Q, R, lane, colbt); break;
        case 4: dp_register_strip<4>(sc, S, Q, R, lane, colbt); break;
        default: dp_shared_strip(sc, S, Q, R, lane, colbt); break;
        }
        const uint32_t last_lane = (Q - 1) / T;
        const bt_state bt = backtrace_start<32>(sc, S.sM, S.sD, S.sI, 0, T, Q, R, last_lane, (Q - 1) % T, colbt);

        // ---- traceback: pointer chase by lane 0, one step code per move, written in reverse
        uint32_t nsteps = 0, leading_clip = 0, beginPos = 0;
        const uint32_t trailing_clip = (bt.queryBegin < Q) ? (Q - bt.queryBegin) : 0;
        if (lane == 0)
        {
            uint32_t qb = bt.queryBegin, rb = bt.refBegin;
            uint32_t idx = qb * W + rb;
            int state = bt.state;
            while (true)
            {
                // MATCH consumes a query and a reference base, DELETE a reference base, INSERT a query base; the walk ends when the
                // state would consume past an edge (SingleRefAlignerSharedImpl.hh:124-146)
                const uint32_t pv = S.ptr[idx];
                const uint32_t dq = state != ST_DELETE, dr = state != ST_INSERT;
                if ((dq && qb == 0) || (dr && rb == 0)) break;
                qb -= dq;
                rb -= dr;
                idx -= dq * W + dr;
                S.steps[nsteps++] = static_cast<uint8_t>(state);
                state = (pv >> (2 * state)) & 3;
            }
            leading_clip = qb;
            beginPos = rb;
        }
        nsteps = __shfl_sync(FULL, nsteps, 0);
        leading_clip = __shfl_sync(FULL, leading_clip, 0);
        beginPos = __shfl_sync(FULL, beginPos, 0);
        __syncwarp();

        // ---- forward emission by the whole warp: op type per step (M split into '='/'X', 'N' on either side is a mismatch),
        //      run boundaries by comparing with the previous step, run index by ballot/popc scan, run length from the next boundary
        uint32_t* cg = cigar + static_cast<size_t>(prob) * max_ops;
        uint32_t n_ops = 0;
        if (leading_clip)
        {
            if (lane == 0 && n_ops < max_ops) cg[n_ops] = (leading_clip << 4) | CIG_S;
            ++n_ops;
        }
        {
            uint32_t qi_base = leading_clip, ri_base = beginPos; // query/ref index at the first step of the current block of 32 steps
            int prev_type = -1;                                   // op type of the last step of the previous block
            uint32_t run_start = 0;                               // forward step index where the open run began
            int run_type = -1;
            for (uint32_t b = 0; b < nsteps; b += 32)
            {
                const uint32_t f = b + lane; // forward step index
                const bool valid = f < nsteps;
                const int st = valid ? S.steps[nsteps - 1 - f] : -1;
                const uint32_t consumes_q = valid && (st == ST_MATCH || st == ST_INSERT);
                const uint32_t consumes_r = valid && (st == ST_MATCH || st == ST_DELETE);
                const uint32_t mq = __ballot_sync(FULL, consumes_q), mr = __ballot_sync(FULL, consumes_r);
                const uint32_t below = (1u << lane) - 1u;
                const uint32_t qi = qi_base + __popc(mq & below), rix = ri_base + __popc(mr & below);
                int type = -1;
                if (valid)
                {
                    if (st == ST_MATCH)
                    {
                        const char a = S.qs[qi], c = S.rs[rix];
                        type = (a == c && a != 'N' && c != 'N') ? CIG_EQ : CIG_X;
                    }
                    else type = (st == ST_DELETE) ? CIG_D : CIG_I;
                }
                int before = __shfl_up_sync(FULL, type, 1);
                if (lane == 0) before = prev_type;
                const bool is_start = valid && (type != before);
                const uint32_t ms = __ballot_sync(FULL, is_start);
                // close the run left open by the previous block(s) if this block starts a new one, then emit the runs that both
                // start and end inside this block; the last run of the block stays open
                if (ms)
                {
                    const uint32_t first = __ffs(ms) - 1;
                    if (run_type >= 0)
                    {
                        if (lane == 0 && n_ops < max_ops) cg[n_ops] = ((b + first - run_start) << 4) | static_cast<uint32_t>(run_type);
                        ++n_ops;
                    }
                    if (is_start)
                    {
                        const uint32_t higher = ms & ~((2u << lane) - 1u); // run starts after this lane
                        if (higher)
                        {
                            const uint32_t nxt = __ffs(higher) - 1;
                            const uint32_t slot_i = n_ops + __popc(ms & below);
                            if (slot_i < max_ops) cg[slot_i] = ((nxt - lane) << 4) | static_cast<uint32_t>(type);
                        }
                    }
                    const uint32_t lastst = 31 - __clz(ms);
                    n_ops += __popc(ms) - 1;
                    run_start = b + lastst;
                    run_type = __shfl_sync(FULL, type, lastst);
                }
                const uint32_t nvalid = min(32u, nsteps - b);
                prev_type = __shfl_sync(FULL, type, nvalid - 1);
                qi_base += __popc(mq);
                ri_base += __popc(mr);
            }
            if (run_type >= 0)
            {
                if (lane == 0 && n_ops < max_ops) cg[n_ops] = ((nsteps - run_start) << 4) | static_cast<uint32_t>(run_type);
                ++n_ops;
            }
        }
        if (trailing_clip)
        {
            if (lane == 0 && n_ops < max_ops) cg[n_ops] = (trailing_clip << 4) | CIG_S;
            ++n_ops;
        }
        if (lane == 0)
        {
            res[prob].score = bt.max;
            res[prob].beginPos = static_cast<int>(beginPos);
            res[prob].n_ops = n_ops;
            res[prob].status = n_ops > max_ops ? 1u : 0u;
        }
        __syncwarp();
    }
}

} // namespace

// K3's launcher.  It counts 4 launches whatever ran, the count sx_global_align_dev has always reported.
int sx_k3_run(sx_ctx* ctx, const sx_ga_scores* sc, const sx_ga_batch* d, sx_ga_result* res_dev, uint32_t* cigar_dev, unsigned* launches)
{
    // small matrices (the common case: haplotypes of an active region) run in 8-lane groups; what is left comes back as a list
    const uint32_t* large = nullptr;
    uint32_t n_large = 0, need = 0;
    int rc = sx_k3_group_launch(ctx, sc, d, res_dev, cigar_dev, &large, &n_large, &need);
    if (rc) return rc;
    if (n_large)
    {
        // one warp per matrix, one shared-memory slot per warp; problems that do not fit a slot report status 2
        size_t slot = (need + 15u) & ~size_t(15);
        int warps = K3_WARPS;
        while (warps > 1 && slot * warps > ctx->smem_optin) warps >>= 1; // very large matrices: fewer warps per CTA
        slot = std::min(slot, ctx->smem_optin & ~size_t(15));
        const size_t smem = slot * warps;
        if (smem > 48 * 1024) SX_CUDA(ctx, cudaFuncSetAttribute(k3_global_align_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(ctx->smem_optin)));
        const int grid = static_cast<int>(std::min<uint32_t>((n_large + warps - 1) / warps, (uint32_t)ctx->sm_count * 16));
        k3_global_align_kernel<<<grid, warps * 32, smem, ctx->s_compute>>>(d->query, d->ref, d->query_off, d->ref_off, n_large, d->max_ops, *sc, res_dev, cigar_dev, (uint32_t)slot,
                                                                         large);
        SX_CUDA(ctx, cudaGetLastError());
    }
    *launches += 4;
    return SX_OK;
}

extern "C" int sx_global_align_dev(sx_ctx* ctx, const sx_ga_scores* sc, const sx_ga_batch* d, sx_ga_result* res_dev, uint32_t* cigar_dev)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    if (!sc || !d || !res_dev || !cigar_dev) return sx_fail(ctx, SX_ERR_ARG, "sx_global_align_dev: NULL argument");
    if (d->n == 0) return SX_OK;
    return sx_run_timed(ctx, [&](unsigned* launches) { return sx_k3_run(ctx, sc, d, res_dev, cigar_dev, launches); });
}

extern "C" int sx_global_align(sx_ctx* ctx, const sx_ga_scores* sc, const sx_ga_batch* b, sx_ga_result* res_host, uint32_t* cigar_host)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    if (!sc || !b || !res_host || !cigar_host || !b->query_off || !b->ref_off) return sx_fail(ctx, SX_ERR_ARG, "sx_global_align: NULL argument");
    if (b->n == 0) return SX_OK;
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    for (uint32_t i = 0; i < b->n; ++i)
    {
        const uint32_t Q = b->query_off[i + 1] - b->query_off[i], R = b->ref_off[i + 1] - b->ref_off[i];
        if (Q == 0 || R == 0) return sx_fail(ctx, SX_ERR_ARG, "sx_global_align: empty query or reference in problem %u (asserted at GlobalAlignerImpl.hh:47-48)", i);
    }
    sx_call_timer t(ctx);
    sx_ga_batch d = *b;
    int rc;
    if ((rc = sx_upload(ctx, sx_host_slot(9), b->query, b->query_off[b->n], d.query, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(10), b->ref, b->ref_off[b->n], d.ref, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(11), b->query_off, (size_t)b->n + 1, d.query_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(12), b->ref_off, (size_t)b->n + 1, d.ref_off, 16))) return rc;
    sx_ga_result* d_res = nullptr;
    uint32_t* d_cig = nullptr;
    if ((rc = sx_take(ctx, sx_host_slot(13), b->n, d_res, 0))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(14), (size_t)b->n * b->max_ops, d_cig, 16))) return rc;
    SX_CUDA(ctx, cudaMemsetAsync(d_cig, 0, (size_t)b->n * b->max_ops * 4, ctx->s_compute)); // unused cigar slots read as 0
    unsigned device_entry_count = 0; // (the launcher counts what sx_global_align_dev reports; this entry has always reported one launch)
    if ((rc = sx_k3_run(ctx, sc, &d, d_res, d_cig, &device_entry_count))) return rc;
    if ((rc = sx_download(ctx, res_host, d_res, b->n))) return rc;
    if ((rc = sx_download(ctx, cigar_host, d_cig, (size_t)b->n * b->max_ops))) return rc;
    return t.finish(1);
}
