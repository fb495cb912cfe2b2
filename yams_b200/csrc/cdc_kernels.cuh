// cdc_kernels.cuh -- kernel argument blocks and declarations shared by cdc.cu / sha256.cu / ingest.cu
#pragma once
#include "cdc_logic.h"
#include "common.cuh"

namespace yb {

struct ScanArgs {
    const uint8_t* data;   // data[0] is stream position base_pos
    uint64_t base_pos;
    uint64_t lowest;       // lowest readable stream position
    uint64_t origin;       // tile origin: <= scan_lo, address of `origin` is 16-byte aligned
    uint64_t scan_lo;      // first stream position to test
    uint64_t scan_hi;      // one past the last stream position to test
    const uint64_t* table; // 256 x u64 (device)
    CdcParams P;
};

// Cut selection over a layout of files (cdc_logic.h): one streaming feed, or many independent streams ("files") in ONE
// device buffer, where every file start is preceded by >= 64 zero bytes, so the rolling hash of the buffer equals the
// hash of the file alone (the reference's ring buffer starts zeroed, chunker.h:150-154).
struct BatchArgs {
    BatchLayout L;            // candidates + file layout (cdc_logic.h)
    CdcParams P;
};

__global__ void batch_next_kernel(BatchArgs B, uint64_t* npos, uint32_t* next, uint32_t* forced, uint32_t* cnt);
__global__ void batch_mask_counts_kernel(const uint8_t* onchain, uint32_t* cnt, uint32_t nnodes);
__global__ void batch_emit_kernel(BatchArgs B, const uint64_t* npos, const uint32_t* next, const uint32_t* forced,
                                  const uint8_t* onchain, const uint32_t* offsets, yams_chunk_desc* out, uint64_t* open_start);
__global__ void batch_first_kernel(BatchArgs B, const uint32_t* offsets, const uint64_t* total, uint64_t* first);
__global__ void batch_rebase_kernel(BatchArgs B, yams_chunk_desc* descs, uint64_t n);

__global__ void cdc_count_kernel(ScanArgs A, uint32_t ntiles, uint32_t* tile_counts);
__global__ void cdc_write_kernel(ScanArgs A, uint32_t ntiles, const uint32_t* tile_counts,
                                 const uint32_t* tile_offsets, uint64_t* cand);
__global__ void cdc_exit_kernel(const uint32_t* next, uint32_t nnodes, uint32_t* exit_out);
__global__ void cdc_walk_kernel(const uint32_t* exit_in, uint32_t nnodes, uint32_t* entry);
__global__ void cdc_mark_kernel(const uint32_t* next, uint32_t nnodes, const uint32_t* entry, uint8_t* onchain);

constexpr int kScanThreads = 256;
constexpr int kScanIters = 4;                                     // 16-byte loads per thread per tile
constexpr uint32_t kTileBytes = kScanThreads * 16 * kScanIters;   // 16 KiB

// single-pass candidate scan (cdc.cu); SC_TILE must divide the tile grid used by the two-pass kernels
constexpr uint32_t kSinglePassTile = 4096;
constexpr uint32_t kSinglePassWarpsPerCta = 16;
yams_status_t launch_scan_single_pass(const ScanArgs& A, uint32_t ntiles, uint64_t* cand_tmp, uint32_t* slice_counts,
                                      uint32_t slice_cap, uint32_t nslices, uint64_t* cand, uint64_t* scalars, cudaStream_t st);

yams_status_t resolve_params(const yams_cdc_config* cfg, CdcParams* P, uint64_t table[256]);
yams_status_t launch_sha256_chunks(const uint8_t* d_data, uint64_t base_pos, yams_chunk_desc* d_descs,
                                   uint32_t first, uint32_t n, unsigned int* d_counter, int sm_count,
                                   cudaStream_t st, uint32_t* d_order_ws, uint64_t total_bytes);
// workspace of the longest-first order: 64 counters + one index per chunk
inline size_t sha256_order_ws_bytes(uint64_t n) { return (size_t)(n + 64) * sizeof(uint32_t); }
yams_status_t launch_dedup_stats(const yams_chunk_desc* d_descs, uint32_t n, uint32_t* d_table, uint64_t slots,
                                 unsigned long long* d_out, cudaStream_t st);
yams_status_t launch_synth_bytes(uint64_t seed, uint64_t start, uint64_t n, uint8_t* d_out, int sm_count,
                                 cudaStream_t st);

}  // namespace yb
