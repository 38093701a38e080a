// k3_common.cuh -- pieces shared by the two GlobalAligner kernels (k3_global_align.cu: one warp per matrix; k3_group.cu: one
// 8-lane group per matrix).  Semantics follow /root/reference/src/c++/lib/alignment/ (AlignerBase.hh:71-92, AlignerUtil.hh:47-80).
#pragma once

#include "sx_internal.h"

#include <climits>

namespace k3
{
constexpr unsigned FULL = 0xffffffffu;
constexpr int BAD = -10000; // badVal, GlobalAlignerImpl.hh:58
enum { ST_MATCH = 0, ST_DELETE = 1, ST_INSERT = 2 };
enum { CIG_M = 0, CIG_I = 1, CIG_D = 2, CIG_S = 4, CIG_EQ = 7, CIG_X = 8 };

// first-argument-wins maximum of three with the index of the winner (AlignerBase::max3)
__device__ __forceinline__ uint32_t max3(int& mx, int v0, int v1, int v2)
{
    mx = v0;
    uint32_t p = 0;
    if (v1 > v0)
    {
        mx = v1;
        p = 1;
    }
    if (v2 > mx)
    {
        mx = v2;
        p = 2;
    }
    return p;
}

struct bt_state // BackTrace<int>
{
    int max;
    int state;
    uint32_t queryBegin, refBegin;
    bool isInit;
};
__device__ __forceinline__ void update_bt(bt_state& b, int v, uint32_t refIndex, uint32_t queryIndex, int state)
{
    if (!b.isInit || v > b.max)
    {
        b.max = v;
        b.refBegin = refIndex;
        b.queryBegin = queryIndex;
        b.isInit = true;
        b.state = state;
    }
}

// scores of DP row 0 at matrix column c >= 1 (GlobalAlignerImpl.hh:104-126) and of the initial column at DP row `row` (:69-88)
__device__ __forceinline__ void row0_scores(const sx_ga_scores& sc, int c, int& m, int& d, int& i)
{
    m = sc.isRequireEdgeDeletion ? BAD : 0;
    d = sc.isRequireEdgeDeletion ? sc.open + c * sc.extend : BAD;
    i = BAD;
}
__device__ __forceinline__ void col0_scores(const sx_ga_scores& sc, int row, int& m, int& d, int& i)
{
    m = row * sc.offEdge;
    d = BAD;
    i = sc.isAllowEdgeInsertion ? sc.open + row * sc.extend : BAD;
}
__host__ __device__ __forceinline__ uint32_t pad16u(uint32_t x) { return (x + 15u) & ~15u; }

// The warp kernel's per-warp shared-memory slot for a (Q, R) problem: byte offsets of its regions (the pointer matrix is at 0) and its
// size.  The size decides status 2, so the kernel's carving and the host's launch sizing both read it from here.
struct k3_slot_layout
{
    uint32_t strips, query, ref, steps, bytes;
};
__host__ __device__ __forceinline__ k3_slot_layout k3_slot(uint32_t Q, uint32_t R)
{
    const uint32_t T = (Q + 31) / 32;
    k3_slot_layout s;
    uint32_t o = 0;
    o += pad16u((Q + 1) * (R + 1)); // pointer matrix
    s.strips = o;
    o += 3u * 32u * T * 4u; // final-column score strips (and the working strips of the long-query fallback)
    s.query = o;
    o += pad16u(Q + 8);
    s.ref = o;
    o += pad16u(R + 8);
    s.steps = o;
    o += pad16u(Q + R + 8); // traceback steps
    s.bytes = o;
    return s;
}
__host__ __device__ __forceinline__ uint32_t k3_slot_bytes(uint32_t Q, uint32_t R) { return k3_slot(Q, R).bytes; }

// The backtrace start (GlobalAlignerImpl.hh:178-209) of the matrix on lanes gbase .. gbase + G - 1, in the reference's candidate order
// with strict '>' updates.  Lane gbase + l owns query rows l*T .. l*T + T - 1, and the final-column scores of row r of its strip are at
// [r * 32 + gbase + l] of sM, sD and sI.  DP row Q is strip row r_last of lane gbase + last_lane, whose colbt holds that row's match
// candidates (:170-175).
template <int G>
__device__ __forceinline__ bt_state backtrace_start(const sx_ga_scores& sc, const int* sM, const int* sD, const int* sI, uint32_t gbase, uint32_t T, uint32_t Q,
                                                    uint32_t R, uint32_t last_lane, uint32_t r_last, const bt_state& colbt)
{
    const uint32_t gl = (threadIdx.x & 31) & (G - 1);
    bt_state bt;
    bt.max = __shfl_sync(FULL, colbt.max, gbase + last_lane);
    bt.refBegin = __shfl_sync(FULL, colbt.refBegin, gbase + last_lane);
    bt.isInit = __shfl_sync(FULL, colbt.isInit ? 1 : 0, gbase + last_lane) != 0;
    bt.queryBegin = Q;
    bt.state = ST_MATCH;
    const uint32_t lastIdx = r_last * 32 + gbase + last_lane;
    if (sc.isRequireEdgeDeletion)
    {
        update_bt(bt, sM[lastIdx], R, Q, ST_MATCH);
        update_bt(bt, sD[lastIdx], R, Q, ST_DELETE);
    }
    if (sc.isAllowEdgeInsertion) update_bt(bt, sI[lastIdx], R, Q, ST_INSERT);
    // query falls off the end of the reference: candidates for queryIndex 0..Q-1 in increasing order == the maximum value with the
    // smallest queryIndex
    int best = INT_MIN;
    uint32_t besti = 0xffffffffu;
    for (uint32_t queryIndex = gl; queryIndex < Q; queryIndex += G)
    {
        int mval;
        if (queryIndex == 0) mval = sc.isRequireEdgeDeletion ? BAD : 0; // DP row 0 at the last column
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
    for (int d = G / 2; d; d >>= 1)
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
    return bt;
}

} // namespace k3

// k3_group.cu: classifies the batch, runs every matrix with Q <= 128 and R <= 255 in 8-lane groups, and returns the list of the
// remaining (large) problems for the warp-per-matrix kernel.
int sx_k3_group_run(sx_ctx* ctx, const sx_ga_scores* sc, const sx_ga_batch* d, sx_ga_result* res_dev, uint32_t* cigar_dev, const uint32_t** large_order_dev,
                    uint32_t* n_large, uint32_t* large_slot_need);
