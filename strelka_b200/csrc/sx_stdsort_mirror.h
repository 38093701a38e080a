// sx_stdsort_mirror.h -- restatement of libstdc++'s std::sort (bits/stl_algo.h: __introsort_loop with
// _S_threshold = 16, median-of-three to first, unguarded Hoare partition, heap-sort fallback at depth
// 2*floor(log2(n)), then __final_insertion_sort), specialised to sorting an index array by DESCENDING key.
//
// Why it exists: the reference sorts each (strand x base) group of a pileup with
//     std::sort(ic.begin(), ic.end(), sort_icall_by_eprob(pi))      blt_common/adjust_joint_eprob.cpp:149
// whose comparator looks only at the 6-bit quality, and then hands the k-th element of the sorted order the
// k-th dependency exponent.  std::sort is not stable, so WHICH of several equal-quality calls receives which
// exponent -- and with it the order of the float additions in get_diploid_gt_lhood -- is decided by the exact
// sequence of swaps libstdc++ performs.  Reproducing the integer PL fields bit-for-bit therefore means
// reproducing that permutation.  For n <= 16 the algorithm degenerates to a (stable) insertion sort; the
// partitioning path matters for deeper groups.  tests/test_stdsort_mirror.py fuzzes this against the real
// std::sort (oracle: ox_sort_std).
#pragma once

#include <stdint.h>

#ifndef SX_HD
#if defined(__CUDACC__)
#define SX_HD __device__ __forceinline__
#else
#define SX_HD static inline
#endif
#endif

#define SX_SORT_COMP(a, b) (key[(a)] > key[(b)]) /* sort_icall_by_eprob::operator() */

template <typename IdxT, typename KeyT> SX_HD void sx_sort_unguarded_linear_insert(IdxT* v, int last, const KeyT& key)
{
    const IdxT val = v[last];
    int next = last - 1;
    while (SX_SORT_COMP(val, v[next]))
    {
        v[last] = v[next];
        last = next;
        --next;
    }
    v[last] = val;
}

template <typename IdxT, typename KeyT> SX_HD void sx_sort_insertion(IdxT* v, int first, int last, const KeyT& key)
{
    if (first == last) return;
    for (int i = first + 1; i != last; ++i)
    {
        if (SX_SORT_COMP(v[i], v[first]))
        {
            const IdxT val = v[i];
            for (int j = i; j > first; --j) v[j] = v[j - 1]; // move_backward(first, i, i+1)
            v[first] = val;
        }
        else
        {
            sx_sort_unguarded_linear_insert(v, i, key);
        }
    }
}

template <typename IdxT, typename KeyT> SX_HD void sx_sort_push_heap(IdxT* v, int first, int holeIndex, int topIndex, IdxT value, const KeyT& key)
{
    int parent = (holeIndex - 1) / 2;
    while (holeIndex > topIndex && SX_SORT_COMP(v[first + parent], value))
    {
        v[first + holeIndex] = v[first + parent];
        holeIndex = parent;
        parent = (holeIndex - 1) / 2;
    }
    v[first + holeIndex] = value;
}

template <typename IdxT, typename KeyT> SX_HD void sx_sort_adjust_heap(IdxT* v, int first, int holeIndex, int len, IdxT value, const KeyT& key)
{
    const int topIndex = holeIndex;
    int secondChild = holeIndex;
    while (secondChild < (len - 1) / 2)
    {
        secondChild = 2 * (secondChild + 1);
        if (SX_SORT_COMP(v[first + secondChild], v[first + (secondChild - 1)])) secondChild--;
        v[first + holeIndex] = v[first + secondChild];
        holeIndex = secondChild;
    }
    if ((len & 1) == 0 && secondChild == (len - 2) / 2)
    {
        secondChild = 2 * (secondChild + 1);
        v[first + holeIndex] = v[first + (secondChild - 1)];
        holeIndex = secondChild - 1;
    }
    sx_sort_push_heap(v, first, holeIndex, topIndex, value, key);
}

// std::__partial_sort(first, last, last): __heap_select degenerates to make_heap, then sort_heap
template <typename IdxT, typename KeyT> SX_HD void sx_sort_heapsort(IdxT* v, int first, int last, const KeyT& key)
{
    const int len = last - first;
    if (len >= 2)
    {
        int parent = (len - 2) / 2;
        while (true)
        {
            const IdxT value = v[first + parent];
            sx_sort_adjust_heap(v, first, parent, len, value, key);
            if (parent == 0) break;
            parent--;
        }
    }
    while (last - first > 1)
    {
        --last;
        const IdxT value = v[last]; // __pop_heap(first, last, last)
        v[last] = v[first];
        sx_sort_adjust_heap(v, first, 0, last - first, value, key);
    }
}

// StackN bounds the explicit stack: every partition pushes one entry and spends one unit of depth_limit = 2*floor(log2(n)), so
// 2*floor(log2(n_max)) + 1 entries cover every n <= n_max (64 covers any 32-bit n; 16 covers n < 256).
// __introsort_loop alone (n > 16).  What std::sort does after it, __final_insertion_sort, is an insertion sort, and an insertion sort is
// stable: the final order is the stable descending sort of the array this leaves.  A caller that needs only part of that order (the first
// few positions) can take it from here without the insertion sort.
template <int StackN = 64, typename IdxT, typename KeyT> SX_HD void sx_introsort_loop_desc(IdxT* v, const int n, const KeyT& key)
{
    // recursion on the right part replaced by an explicit stack
    int stack_first[StackN], stack_last[StackN], stack_depth[StackN];
    int sp = 0;
    int lg = 0;
    for (int t = n; t > 1; t >>= 1) ++lg; // std::__lg
    stack_first[0] = 0;
    stack_last[0] = n;
    stack_depth[0] = lg * 2;
    sp = 1;
    while (sp > 0)
    {
        --sp;
        const int first = stack_first[sp];
        int last = stack_last[sp];
        int depth_limit = stack_depth[sp];
        while (last - first > 16)
        {
            if (depth_limit == 0)
            {
                sx_sort_heapsort(v, first, last, key);
                break;
            }
            --depth_limit;
            // __unguarded_partition_pivot
            const int mid = first + (last - first) / 2;
            {
                // __move_median_to_first(result=first, a=first+1, b=mid, c=last-1)
                const int a = first + 1, b = mid, c = last - 1;
                int m;
                if (SX_SORT_COMP(v[a], v[b]))
                {
                    if (SX_SORT_COMP(v[b], v[c])) m = b;
                    else if (SX_SORT_COMP(v[a], v[c])) m = c;
                    else m = a;
                }
                else if (SX_SORT_COMP(v[a], v[c])) m = a;
                else if (SX_SORT_COMP(v[b], v[c])) m = c;
                else m = b;
                const IdxT t = v[first];
                v[first] = v[m];
                v[m] = t;
            }
            int lo = first + 1, hi = last;
            const IdxT pivot = v[first]; // the pivot element does not move during the partition
            while (true)
            {
                while (SX_SORT_COMP(v[lo], pivot)) ++lo;
                --hi;
                while (SX_SORT_COMP(pivot, v[hi])) --hi;
                if (!(lo < hi)) break;
                const IdxT t = v[lo];
                v[lo] = v[hi];
                v[hi] = t;
                ++lo;
            }
            const int cut = lo;
            // recurse on [cut, last) first (the reference recursion), continue the loop on [first, cut)
            // ordering between the two sub-ranges does not matter: they are disjoint
            stack_first[sp] = cut;
            stack_last[sp] = last;
            stack_depth[sp] = depth_limit;
            ++sp;
            last = cut;
        }
    }
}

template <int StackN = 64, typename IdxT, typename KeyT> SX_HD void sx_stdsort_desc(IdxT* v, const uint32_t n_, const KeyT& key)
{
    const int n = (int)n_;
    if (n == 0) return;
    if (n <= 16) // __introsort_loop returns at once; __final_insertion_sort is a plain insertion sort
    {
        sx_sort_insertion(v, 0, n, key);
        return;
    }
    sx_introsort_loop_desc<StackN>(v, n, key);
    // __final_insertion_sort (n > 16)
    sx_sort_insertion(v, 0, 16, key);
    for (int i = 16; i != n; ++i) sx_sort_unguarded_linear_insert(v, i, key);
}
