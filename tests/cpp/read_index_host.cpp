// The read index's per-read body (strelka_b200/csrc/sx_read_index.cuh) compiled for the host: the 'N' count of reads at any byte offset and
// length, and the buffer position, for tests/test_read_index.py.
#include "sx_read_index.cuh"

extern "C" void read_index_count_n(const uint8_t* pool, const uint64_t* off, const uint16_t* len, const uint32_t n, uint32_t* out)
{
    for (uint32_t r = 0; r < n; ++r) out[r] = sxi_count_n(pool + off[r], len[r]);
}

extern "C" void read_index_buffer_pos(const int32_t* pos, const uint32_t* seg_off, const sx_aln_seg* segs, const uint32_t n, int32_t* out)
{
    for (uint32_t r = 0; r < n; ++r) out[r] = sxi_buffer_pos(pos[r], segs + seg_off[r], seg_off[r + 1] - seg_off[r]);
}
