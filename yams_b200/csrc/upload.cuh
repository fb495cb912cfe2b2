// upload.cuh -- the pinned, double-buffered upload of many pageable host buffers into one device layout (ingest.cu; DESIGN §3.4).
#pragma once
#include <vector>

#include "common.cuh"

namespace yb {

// One piece of a packed layout: `len` bytes from host memory `src` at layout position `pos`.
struct LayoutPiece {
    uint64_t pos, len;
    const uint8_t* src;
};

// Uploads layout positions [0, total) to d_dst on stream st: the bytes of the pieces (ascending, disjoint), zeros elsewhere.
// Host threads assemble each slice in one of the two pinned buffers `pin` while the previous slice is on the wire;
// pin_done[b] (created by the caller) marks the end of the copy out of pin[b].
yams_status_t staged_upload(HostBuf pin[2], cudaEvent_t pin_done[2], uint8_t* d_dst, uint64_t total,
                            const std::vector<LayoutPiece>& pieces, cudaStream_t st);

}  // namespace yb
