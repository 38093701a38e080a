// k3_group.cu -- K3 for SMALL matrices (Q <= 128, R <= 255; the haplotypes of an active region): one 8-lane GROUP per DP matrix,
// four matrices per warp.
//
// Same anti-diagonal wavefront as k3_global_align.cu -- each lane owns a strip of consecutive query rows in registers, the scores of
// the row above / the diagonal cross lanes by __shfl_up (width 8) -- but with strips of T = ceil(Q/8) rows instead of ceil(Q/32):
// for a 70 x 65 matrix that is 7 fill/drain steps instead of 22, 9 cells of work per shuffle round instead of 3, and 93 % of the
// lane-rows are real cells instead of 70 %.
//
// T is a template parameter (1..16), so the batch is bucketed by (T, reference-length class) on the device first and each T gets its
// own launch over its bucket; the four matrices of a warp therefore share T and have similar R.
//
// The 3 x 2-bit back pointers of cell (row, col) are stored at  scratch[warp][(t * T + r) * 32 + lane]  with t = col + lane-in-group
// the wavefront step, r the row within the lane's strip: every warp store is one coalesced 32-byte sector.  The scratch of the resident
// warps is tens of MB; on an H100 (50 MB of L2) the larger buckets' scratch does not all stay in the L2, so part of the traceback reads
// come from HBM (K3 is still about 1 % of a cfg2 step there, README.md).  The pointer chase of the traceback reads it back by the same mapping;
// traceback and '='/'X' expansion run on lane 0 of each group (four at a time per warp).
// Arithmetic, max3 tie rule and candidate order are those of GlobalAligner<int> (alignment/GlobalAlignerImpl.hh:36-228): bit-exact.
#include "k3_common.cuh"

#include <algorithm>
#include <climits>

namespace
{
using namespace k3;

constexpr uint32_t KG_MAX_Q = 128, KG_MAX_R = 255;
constexpr int KG_WARPS = 4;       // warps per CTA
constexpr int KG_G = 8;           // lanes per matrix
constexpr int KG_RCLASSES = 4;    // reference-length classes per T (R/64)
constexpr int KG_BUCKETS = 16 * KG_RCLASSES + 1; // + 1: large problems (warp kernel)

struct kg_info
{
    uint32_t hist[KG_BUCKETS];
    uint32_t max_r[16];  // per T class
    uint32_t large_need; // shared-memory slot of the largest "large" problem
    uint32_t work[16];   // per T class: next quad to hand out (kg_align_kernel)
};

__device__ __forceinline__ uint32_t kg_bucket(uint32_t Q, uint32_t R, uint32_t max_q)
{
    if (Q == 0 || R == 0 || Q > max_q || R > KG_MAX_R) return KG_BUCKETS - 1;
    const uint32_t T = (Q + KG_G - 1) / KG_G;
    return (T - 1) * KG_RCLASSES + min((uint32_t)KG_RCLASSES - 1, R >> 6);
}

__global__ void kg_classify_kernel(const uint32_t* __restrict__ query_off, const uint32_t* __restrict__ ref_off, uint32_t n, kg_info* __restrict__ info,
                                   uint32_t max_q)
{
    __shared__ uint32_t h[KG_BUCKETS];
    __shared__ uint32_t mr[16];
    __shared__ uint32_t need;
    for (int i = threadIdx.x; i < KG_BUCKETS; i += blockDim.x) h[i] = 0;
    if (threadIdx.x < 16) mr[threadIdx.x] = 0;
    if (threadIdx.x == 0) need = 0;
    __syncthreads();
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    {
        const uint32_t Q = query_off[i + 1] - query_off[i], R = ref_off[i + 1] - ref_off[i];
        const uint32_t b = kg_bucket(Q, R, max_q);
        atomicAdd(&h[b], 1u);
        if (b == KG_BUCKETS - 1)
        {
            if (Q && R) atomicMax(&need, k3_slot_bytes(Q, R));
        }
        else atomicMax(&mr[b / KG_RCLASSES], R);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < KG_BUCKETS; i += blockDim.x)
        if (h[i]) atomicAdd(&info->hist[i], h[i]);
    if (threadIdx.x < 16 && mr[threadIdx.x]) atomicMax(&info->max_r[threadIdx.x], mr[threadIdx.x]);
    if (threadIdx.x == 0 && need) atomicMax(&info->large_need, need);
}

__global__ void kg_scatter_kernel(const uint32_t* __restrict__ query_off, const uint32_t* __restrict__ ref_off, uint32_t n, uint32_t* __restrict__ cursor,
                                  uint32_t* __restrict__ order, uint32_t max_q)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    {
        const uint32_t b = kg_bucket(query_off[i + 1] - query_off[i], ref_off[i + 1] - ref_off[i], max_q);
        order[atomicAdd(&cursor[b], 1u)] = i;
    }
}

constexpr int KG_B = 8; // quads whose DP a warp finishes before it traces back their 4 * KG_B matrices, one per lane
constexpr uint32_t KG_SAVE_WORDS = 6; // per-matrix state kept from the DP to the traceback

// per-warp shared memory: final-column score strips [3][T][32] ints, per group: query (T*8), reference (max_r); the saved start states
template <int T> __host__ __device__ constexpr uint32_t kg_warp_smem(uint32_t max_r)
{
    return 3u * T * 32u * 4u + 4u * (((T * KG_G + 15u) & ~15u) + ((max_r + 15u) & ~15u)) + KG_SAVE_WORDS * 32u * 4u;
}

// Score keys: 64*score + tag, tag = 21 * (3 - state) = the 2-bit code (3 - state) replicated into three 2-bit fields (match 0b111111,
// delete 0b101010, insert 0b010101).  See the comment in kg_align_kernel.
constexpr int KG_KEY_SHIFT = 6;
__device__ __forceinline__ int key_of(int score, int state) { return score * (1 << KG_KEY_SHIFT) + 21 * (3 - state); }
// keeps a loop-invariant constant in its register: without it the compiler folds "cond ? 64*a+63 : 64*b+63" back into per-cell
// multiply-adds on the raw parameters
__device__ __forceinline__ int opaque(int x)
{
    asm volatile("" : "+r"(x));
    return x;
}

template <int T>
__global__ void __launch_bounds__(KG_WARPS * 32) kg_align_kernel(const char* __restrict__ query_pool, const char* __restrict__ ref_pool,
                                                                 const uint32_t* __restrict__ query_off, const uint32_t* __restrict__ ref_off,
                                                                 const uint32_t* __restrict__ order, uint32_t n, uint32_t max_ops, sx_ga_scores sc,
                                                                 sx_ga_result* __restrict__ res, uint32_t* __restrict__ cigar, uint32_t max_r,
                                                                 unsigned char* __restrict__ scratch, size_t scratch_slot, uint32_t* __restrict__ work)
{
    extern __shared__ __align__(16) unsigned char smem[];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t grp = lane >> 3, gl = lane & 7u;
    unsigned char* wsm = smem + (size_t)warp * kg_warp_smem<T>(max_r);
    int* sM = reinterpret_cast<int*>(wsm);
    int* sD = sM + T * 32;
    int* sI = sD + T * 32;
    const uint32_t qpad = (T * KG_G + 15u) & ~15u, rpad = (max_r + 15u) & ~15u;
    unsigned char* gsm = wsm + 3u * T * 32u * 4u + grp * (qpad + rpad);
    char* qs = reinterpret_cast<char*>(gsm);
    char* rs = qs + qpad;
    // start states of the warp's pending matrices (slot = quad-in-batch * 4 + group): prob, Q, queryBegin, refBegin, state, score
    uint32_t* sv = reinterpret_cast<uint32_t*>(wsm + 3u * T * 32u * 4u + 4u * (qpad + rpad));
    const uint32_t gwarp = blockIdx.x * KG_WARPS + warp;
    unsigned char* const wscratch = scratch + (size_t)gwarp * scratch_slot * KG_B;

    const int s_match = sc.match, s_mismatch = sc.mismatch, s_open = sc.open, s_extend = sc.extend, s_insdel = sc.insertDelete;
    const bool req_del = sc.isRequireEdgeDeletion != 0, allow_ins = sc.isAllowEdgeInsertion != 0;
    const int row0M = req_del ? BAD : 0;
    // initial-column / initial-row back pointers, in the stored tag encoding (tag = 3 - state)
    const uint32_t ptr_c0 = (3u - ST_MATCH) | ((3u - ST_MATCH) << 2) | ((3u - (allow_ins ? ST_INSERT : ST_MATCH)) << 4);
    const uint32_t ptr_r0 = (3u - ST_MATCH) | ((3u - (req_del ? ST_DELETE : ST_MATCH)) << 2) | ((3u - ST_MATCH) << 4);
    const int o4 = opaque(s_open * 64), e4 = s_extend * 64, id4 = opaque(s_insdel * 64);
    // addends that also re-tag a winner whose tag bits were cleared
    const int ma4t = opaque(s_match * 64 + 63), mi4t = opaque(s_mismatch * 64 + 63), e4tD = opaque(e4 + 42), e4tI = opaque(e4 + 21);
    const int kRow0M = key_of(row0M, ST_MATCH), kBadD = opaque(key_of(BAD, ST_DELETE)), kBadI = key_of(BAD, ST_INSERT), kDel0 = key_of(s_open, ST_DELETE);
    const bool is_lane0 = gl == 0;
    const uint32_t row0 = gl * T; // query index of this lane's first row

    const uint32_t n_quads = (n + 3) / 4;
    // Quads are handed out one at a time through an atomic counter (so the tail of a launch is one quad, not one batch); a warp runs
    // the DP of up to KG_B quads, keeping their back pointers in KG_B scratch slots, and then traces all of them back at once.
    uint32_t n_pending = 0;
    for (;;)
    {
        uint32_t quad = 0;
        if (lane == 0) quad = atomicAdd(work, 1u);
        quad = __shfl_sync(FULL, quad, 0);
        const bool got = quad < n_quads;
        if (got)
        {
        unsigned char* ptr = wscratch + (size_t)n_pending * scratch_slot;
        const uint32_t k = quad * 4 + grp;
        const bool have = k < n;
        const uint32_t prob = have ? order[k] : 0;
        const uint32_t Q = have ? query_off[prob + 1] - query_off[prob] : 0;
        const uint32_t R = have ? ref_off[prob + 1] - ref_off[prob] : 0;
        const uint32_t last_lane = have ? (Q - 1) / T : 0;
        {
            const char* qg = query_pool + (have ? query_off[prob] : 0);
            const char* rg = ref_pool + (have ? ref_off[prob] : 0);
            for (uint32_t i = gl; i < Q; i += KG_G) qs[i] = qg[i];
            for (uint32_t i = gl; i < R; i += KG_G) rs[i] = rg[i];
        }
        __syncwarp();
        // Scores live in registers as KEYS: 64*score + tag (key_of).  The three arguments of every max3 of the recurrence are (a match
        // value, a delete value, an insert value) in that order, so a plain integer max of keys is exactly AlignerBase::max3's "largest
        // value, first argument wins ties", the tag of the winner says which argument won, and the three-way maxima become single
        // VIMNMX3 / VIADDMNMX instructions.  The tag is replicated in three 2-bit fields so the back-pointer byte of a cell is two
        // bit-selects of the three winners (no shifts).  sx_k3_group_run keeps batches whose penalties could overflow 64*score out of
        // this kernel.
        int rM[T], rD[T], rI[T];
        char qc[T];
#pragma unroll
        for (int r = 0; r < T; ++r)
        {
            const uint32_t qi = row0 + r;
            int m, dd, ii;
            col0_scores(sc, (int)qi + 1, m, dd, ii);
            rM[r] = key_of(m, ST_MATCH);
            rD[r] = key_of(dd, ST_DELETE);
            rI[r] = key_of(ii, ST_INSERT);
            qc[r] = qi < Q ? qs[qi] : 0;
        }
        int c0M, c0D, c0I; // initial column at the DP row above this strip
        col0_scores(sc, (int)row0, c0M, c0D, c0I);
        c0M = key_of(c0M, ST_MATCH);
        c0D = key_of(c0D, ST_DELETE);
        c0I = key_of(c0I, ST_INSERT);
        const uint32_t r_last = have ? (Q - 1) - last_lane * T : 0; // strip-relative index of DP row Q in the group's last lane
        // warp-uniform step count: the longest wavefront of the four groups
        uint32_t n_steps = have ? R + last_lane : 0;
        n_steps = max(n_steps, __shfl_xor_sync(FULL, n_steps, 8));
        n_steps = max(n_steps, __shfl_xor_sync(FULL, n_steps, 16));
        bt_state colbt{0, ST_MATCH, 0, 0, false};
        int sendM = 0, sendD = 0, sendI = 0, prevRecvM = 0, prevRecvD = 0, prevRecvI = 0;
        unsigned char* pstep = ptr + lane;
        for (uint32_t t = 0; t < n_steps; ++t)
        {
            const int recvM = __shfl_up_sync(FULL, sendM, 1, KG_G);
            const int recvD = __shfl_up_sync(FULL, sendD, 1, KG_G);
            const int recvI = __shfl_up_sync(FULL, sendI, 1, KG_G);
            const int j = static_cast<int>(t) - static_cast<int>(gl);
            if (have && j >= 0 && j < static_cast<int>(R) && gl <= last_lane)
            {
                const char rc = rs[j];
                const bool j0 = j == 0;
                int upM = is_lane0 ? kRow0M : recvM;
                int upD = is_lane0 ? (req_del ? kDel0 + (j + 1) * e4 : kBadD) : recvD;
                int upI = is_lane0 ? kBadI : recvI;
                int dgM = j0 ? c0M : (is_lane0 ? kRow0M : prevRecvM);
                int dgD = j0 ? c0D : (is_lane0 ? (req_del ? kDel0 + j * e4 : kBadD) : prevRecvD);
                int dgI = j0 ? c0I : (is_lane0 ? kBadI : prevRecvI);
                int mQ = 0;
#pragma unroll
                for (int r = 0; r < T; ++r)
                {
                    const int lfM = rM[r], lfD = rD[r], lfI = rI[r];
                    // match: max3(diag M, diag D, diag I) + match/mismatch
                    const int km = __vimax3_s32(dgM, dgD, dgI);
                    const int m = (km & ~63) + ((qc[r] == rc) ? ma4t : mi4t);
                    // delete: max3(left M + open, left D, left I + insertDelete) + extend
                    const int kd = __viaddmax_s32(lfM, o4, __viaddmax_s32(lfI, id4, lfD));
                    const int d = (kd & ~63) + e4tD; // (column 0: overwritten with badVal below)
                    // insert: max3(up M + open, badVal, up I) + extend
                    const int ki = __viaddmax_s32(upM, o4, max(kBadD, upI));
                    int ins = (ki & ~63) + e4tI;
                    if (r == 0) ins = (row0 == 0) ? kBadI : ins; // queryIndex 0
                    // back pointers: bits 0-1 from the match winner, 2-3 from the delete winner, 4-5 from the insert winner (raw tags,
                    // state = 3 - tag, decoded by the traceback; bits 6-7 are don't-care).  Rows past Q store too: the slot covers them.
                    pstep[r * 32] = static_cast<unsigned char>((km & 3) | (((kd & 0xf) | (ki & ~0xf)) & ~3));
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
                if (j0) // delete state of the first column is badVal (once per lane per matrix)
                {
#pragma unroll
                    for (int r = 0; r < T; ++r) rD[r] = kBadD;
                    upD = kBadD;
                }
                sendM = upM;
                sendD = upD;
                sendI = upI;
                if (gl == last_lane && !req_del) update_bt(colbt, mQ >> KG_KEY_SHIFT, j + 1, Q, ST_MATCH); // :170-175
            }
            prevRecvM = recvM;
            prevRecvD = recvD;
            prevRecvI = recvI;
            pstep += T * 32;
        }
        // final-column scores of every row
#pragma unroll
        for (int r = 0; r < T; ++r)
        {
            sM[r * 32 + lane] = rM[r] >> KG_KEY_SHIFT; // key -> score (arithmetic shift = floor, exact for negative scores too)
            sD[r * 32 + lane] = rD[r] >> KG_KEY_SHIFT;
            sI[r * 32 + lane] = rI[r] >> KG_KEY_SHIFT;
        }
        __syncwarp();
        // ---- backtrace start selection (:178-209)
        const uint32_t gbase = grp * KG_G;
        bt_state bt;
        bt.max = __shfl_sync(FULL, colbt.max, gbase + last_lane);
        bt.refBegin = __shfl_sync(FULL, colbt.refBegin, gbase + last_lane);
        bt.isInit = __shfl_sync(FULL, colbt.isInit ? 1 : 0, gbase + last_lane) != 0;
        bt.queryBegin = Q;
        bt.state = ST_MATCH;
        {
            const uint32_t lastIdx = r_last * 32 + gbase + last_lane;
            if (req_del)
            {
                update_bt(bt, sM[lastIdx], R, Q, ST_MATCH);
                update_bt(bt, sD[lastIdx], R, Q, ST_DELETE);
            }
            if (allow_ins) update_bt(bt, sI[lastIdx], R, Q, ST_INSERT);
            int best = INT_MIN;
            uint32_t besti = 0xffffffffu;
            for (uint32_t queryIndex = gl; queryIndex < Q; queryIndex += KG_G)
            {
                int mval;
                if (queryIndex == 0) mval = row0M; // DP row 0 at the last column
                else
                {
                    const uint32_t qi = queryIndex - 1;
                    mval = sM[(qi % T) * 32 + gbase + (qi / T)];
                }
                const int v = mval + static_cast<int>(Q - queryIndex) * sc.offEdge;
                if (v > best)
                {
                    best = v;
                    besti = queryIndex;
                }
            }
#pragma unroll
            for (int d = 4; d; d >>= 1)
            {
                const int ov = __shfl_xor_sync(FULL, best, d);
                const uint32_t oi = __shfl_xor_sync(FULL, besti, d);
                if (ov > best || (ov == best && oi < besti))
                {
                    best = ov;
                    besti = oi;
                }
            }
            update_bt(bt, best, R, besti, ST_MATCH);
        }
        // ---- keep the start state for the batched traceback
        if (is_lane0)
        {
            uint32_t* s = sv + (n_pending * 4 + grp) * KG_SAVE_WORDS;
            s[0] = have ? prob : 0xffffffffu;
            s[1] = Q;
            s[2] = bt.queryBegin;
            s[3] = bt.refBegin;
            s[4] = static_cast<uint32_t>(bt.state);
            s[5] = static_cast<uint32_t>(bt.max);
        }
        ++n_pending;
        __syncwarp();
        } // got
        if (n_pending == KG_B || (!got && n_pending))
        {
            __syncwarp();
            // ---- traceback + emission: one matrix per lane (4 * n_pending of them).  The path is walked from its end, so the CIGAR is
            // produced last operation first, into a ring over the caller's max_ops slots, and put in order at the end; the ring keeps
            // exactly what the forward emission keeps on overflow (the first max_ops operations).
            const uint32_t* s = sv + lane * KG_SAVE_WORDS;
            const uint32_t prob = lane < n_pending * 4 ? s[0] : 0xffffffffu;
            if (prob != 0xffffffffu)
            {
                const unsigned char* pm = wscratch + (size_t)(lane >> 2) * scratch_slot;
                const uint32_t gbase = (lane & 3u) * KG_G;
                const uint32_t Q = s[1];
                uint32_t qb = s[2], rb = s[3];
                int state = static_cast<int>(s[4]);
                const char* qg = query_pool + query_off[prob];
                const char* rg = ref_pool + ref_off[prob];
                uint32_t* cg = cigar + static_cast<size_t>(prob) * max_ops;
                uint32_t n_ops = 0, wpos = 0;
                auto push = [&](uint32_t type, uint32_t len) {
                    if (max_ops)
                    {
                        cg[wpos] = (len << 4) | type;
                        if (++wpos == max_ops) wpos = 0;
                    }
                    ++n_ops;
                };
                if (qb < Q) push(CIG_S, Q - qb); // trailing soft clip
                int cur_type = -1;
                uint32_t cur_len = 0;
                while (true)
                {
                    uint32_t pv;
                    if (qb == 0 || rb == 0) pv = (rb == 0) ? ptr_c0 : ptr_r0;
                    else
                    {
                        const uint32_t row = qb - 1, ln = row / T, r = row - ln * T, t = (rb - 1) + ln;
                        pv = pm[(static_cast<size_t>(t) * T + r) * 32 + gbase + ln];
                    }
                    const uint32_t dq = state != ST_DELETE, dr = state != ST_INSERT;
                    if ((dq && qb == 0) || (dr && rb == 0)) break;
                    qb -= dq;
                    rb -= dr;
                    int type;
                    if (state == ST_MATCH)
                    {
                        const char a = __ldg(qg + qb), c = __ldg(rg + rb);
                        type = (a == c && a != 'N' && c != 'N') ? CIG_EQ : CIG_X;
                    }
                    else type = (state == ST_DELETE) ? CIG_D : CIG_I;
                    if (type == cur_type) ++cur_len;
                    else
                    {
                        if (cur_type >= 0) push(static_cast<uint32_t>(cur_type), cur_len);
                        cur_type = type;
                        cur_len = 1;
                    }
                    state = 3 - static_cast<int>((pv >> (2 * state)) & 3u);
                }
                if (cur_type >= 0) push(static_cast<uint32_t>(cur_type), cur_len);
                if (qb) push(CIG_S, qb); // leading soft clip
                // ring -> forward order
                auto reverse = [&](uint32_t lo, uint32_t hi) { // [lo, hi)
                    while (lo + 1 < hi)
                    {
                        --hi;
                        const uint32_t tmp = cg[lo];
                        cg[lo] = cg[hi];
                        cg[hi] = tmp;
                        ++lo;
                    }
                };
                if (n_ops <= max_ops) reverse(0, n_ops);
                else
                {
                    // slot of the forward-first operation is p = (n_ops - 1) mod max_ops; forward[f] = ring[(p - f) mod max_ops]
                    const uint32_t p = (wpos + max_ops - 1) % max_ops, sh = max_ops - 1 - p;
                    reverse(0, max_ops);
                    reverse(0, sh);
                    reverse(sh, max_ops);
                    reverse(0, max_ops);
                }
                res[prob].score = static_cast<int>(s[5]);
                res[prob].beginPos = static_cast<int>(rb);
                res[prob].n_ops = n_ops;
                res[prob].status = n_ops > max_ops ? 1u : 0u;
            }
            __syncwarp();
            n_pending = 0;
        }
        if (!got) break;
    }
}

// upper bound on resident CTAs per SM used for the grid and for the scratch sizing (strips of 10+ rows need > 100 registers)
inline int kg_max_ctas_per_sm(int T) { return T >= 10 ? 4 : 8; }

template <int T>
int kg_launch(sx_ctx* ctx, const sx_ga_scores* sc, const sx_ga_batch* d, sx_ga_result* res_dev, uint32_t* cigar_dev, const uint32_t* order, uint32_t n, uint32_t max_r,
              int scratch_slot_id, uint32_t* work_dev)
{
    if (n == 0) return SX_OK;
    const size_t smem = (size_t)kg_warp_smem<T>(max_r) * KG_WARPS;
    const size_t slot = (((size_t)(max_r + KG_G) * T * 32) + 255) & ~size_t(255);
    const uint32_t quads = (n + 3) / 4;
    if (smem > 48 * 1024) SX_CUDA(ctx, cudaFuncSetAttribute(kg_align_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(ctx->smem_optin)));
    // persistent grid: as many CTAs per SM as the instantiation's registers / shared memory allow (4 for the tall strips, more below)
    int occ = 4;
    SX_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kg_align_kernel<T>, KG_WARPS * 32, smem));
    occ = std::max(1, std::min(occ, kg_max_ctas_per_sm(T)));
    const int grid = static_cast<int>(std::min<uint32_t>((quads + KG_WARPS - 1) / KG_WARPS, (uint32_t)(ctx->sm_count * occ)));
    unsigned char* scratch = nullptr;
    int rc = sx_ensure(ctx, scratch_slot_id, slot * KG_B * (size_t)grid * KG_WARPS, reinterpret_cast<void**>(&scratch));
    if (rc) return rc;
    kg_align_kernel<T><<<grid, KG_WARPS * 32, smem, ctx->s_compute>>>(d->query, d->ref, d->query_off, d->ref_off, order, n, d->max_ops, *sc, res_dev, cigar_dev, max_r, scratch,
                                                                     slot, work_dev);
    SX_CUDA(ctx, cudaGetLastError());
    return SX_OK;
}
} // namespace

int sx_k3_group_run(sx_ctx* ctx, const sx_ga_scores* sc, const sx_ga_batch* d, sx_ga_result* res_dev, uint32_t* cigar_dev, const uint32_t** large_order_dev,
                    uint32_t* n_large, uint32_t* large_slot_need)
{
    kg_info* d_info = nullptr;
    uint32_t* d_cursor = nullptr;
    uint32_t* d_order = nullptr;
    int rc;
    if ((rc = sx_ensure(ctx, 20, sizeof(kg_info), reinterpret_cast<void**>(&d_info)))) return rc;
    if ((rc = sx_ensure(ctx, 21, sizeof(uint32_t) * KG_BUCKETS, reinterpret_cast<void**>(&d_cursor)))) return rc;
    if ((rc = sx_ensure(ctx, 22, sizeof(uint32_t) * (size_t)d->n, reinterpret_cast<void**>(&d_order)))) return rc;
    SX_CUDA(ctx, cudaMemsetAsync(d_info, 0, sizeof(kg_info), ctx->s_compute));
    const int cgrid = static_cast<int>(std::min<uint32_t>((d->n + 255) / 256, 1184));
    // the group kernel keeps 64*score in 32 bits: penalties that could overflow it send the whole batch to the warp kernel
    const auto big = [](int v) { return v > 4096 || v < -4096; };
    const uint32_t max_q = (big(sc->match) || big(sc->mismatch) || big(sc->open) || big(sc->extend) || big(sc->offEdge) || big(sc->insertDelete)) ? 0u : KG_MAX_Q;
    kg_classify_kernel<<<cgrid, 256, 0, ctx->s_compute>>>(d->query_off, d->ref_off, d->n, d_info, max_q);
    kg_info info;
    SX_CUDA(ctx, cudaMemcpyAsync(&info, d_info, sizeof(info), cudaMemcpyDeviceToHost, ctx->s_compute));
    SX_CUDA(ctx, cudaStreamSynchronize(ctx->s_compute));
    uint32_t cursor[KG_BUCKETS], begin[KG_BUCKETS + 1];
    uint32_t acc = 0;
    for (int b = 0; b < KG_BUCKETS; ++b)
    {
        cursor[b] = begin[b] = acc;
        acc += info.hist[b];
    }
    begin[KG_BUCKETS] = acc;
    SX_CUDA(ctx, cudaMemcpyAsync(d_cursor, cursor, sizeof(cursor), cudaMemcpyHostToDevice, ctx->s_compute));
    kg_scatter_kernel<<<cgrid, 256, 0, ctx->s_compute>>>(d->query_off, d->ref_off, d->n, d_cursor, d_order, max_q);
    SX_CUDA(ctx, cudaGetLastError());
#define KG_CASE(TT)                                                                                                                           \
    {                                                                                                                                         \
        const uint32_t b0 = begin[(TT - 1) * KG_RCLASSES], b1 = begin[TT * KG_RCLASSES];                                                       \
        if ((rc = kg_launch<TT>(ctx, sc, d, res_dev, cigar_dev, d_order + b0, b1 - b0, info.max_r[TT - 1], 23, &d_info->work[TT - 1]))) return rc; \
    }
    // one launch per strip height; launches on one stream reuse the same scratch arena (sized for the largest so far by sx_ensure,
    // which only ever grows between launches after a stream-ordered free would be unsafe -- so size it once for the worst class)
    {
        size_t worst = 0;
        for (int t = 1; t <= 16; ++t)
            if (begin[t * KG_RCLASSES] > begin[(t - 1) * KG_RCLASSES])
                worst = std::max(worst, (((size_t)(info.max_r[t - 1] + KG_G) * t * 32 + 255) & ~size_t(255)) * kg_max_ctas_per_sm(t));
        void* p = nullptr;
        if (worst && (rc = sx_ensure(ctx, 23, worst * KG_B * (size_t)ctx->sm_count * KG_WARPS, &p))) return rc;
    }
    KG_CASE(1) KG_CASE(2) KG_CASE(3) KG_CASE(4) KG_CASE(5) KG_CASE(6) KG_CASE(7) KG_CASE(8)
    KG_CASE(9) KG_CASE(10) KG_CASE(11) KG_CASE(12) KG_CASE(13) KG_CASE(14) KG_CASE(15) KG_CASE(16)
#undef KG_CASE
    *large_order_dev = d_order + begin[KG_BUCKETS - 1];
    *n_large = info.hist[KG_BUCKETS - 1];
    *large_slot_need = info.large_need;
    return SX_OK;
}
