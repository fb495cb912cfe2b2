// cdc_sim.cpp -- TEST-ONLY host emulation of the GPU chunking pipeline.  It calls the integer logic the kernels call
// (yams_b200/csrc/cdc_logic.h: is_candidate, batch_next, block_exit_seq, block_mark_seq, batch_emit, batch_file_offset)
// in the same order as cdc.cu / ingest.cu, but sequentially on the CPU, so the logic can be checked against the oracle on
// machines without a GPU.  Every chunk's offset and size comes from cdc_logic.h.  Not part of the product; never linked
// into libyams_b200.so.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../yams_b200/csrc/cdc_logic.h"

using namespace yb;

namespace {
struct Params {
    CdcParams P;
    uint64_t T[256];
    bool no_candidates;
};

bool resolve(uint64_t window, uint64_t minc, uint64_t maxc, uint64_t poly, uint64_t mask, int variant, Params* out) {
    // mirrors yb::resolve_params in cdc.cu
    memset(&out->P, 0, sizeof(out->P));
    if (window > (uint64_t)kMaxWindow) return false;
    uint64_t p = poly ? poly : kDefaultPoly;
    for (int b = 0; b < 256; ++b) out->T[b] = table_entry(p, (uint32_t)b);
    out->P.mask = mask;
    out->P.window = window ? (uint32_t)window : 1u;
    out->P.steps = mask_steps(mask);
    uint64_t force = minc > maxc ? minc : maxc;
    if (variant == 0) {
        out->P.lo = (minc > 1 ? minc : 1) - 1;
        if (force == 0) force = 1;
    } else {
        out->P.lo = minc;
        if (force == 0) return false;
    }
    out->P.force = force;
    out->no_candidates = out->P.lo >= out->P.force;
    return true;
}

// candidate positions in [lo, hi), ascending (the candidate scan)
std::vector<uint64_t> candidates(const ByteView& view, const Params& pr, uint64_t lo, uint64_t hi) {
    std::vector<uint64_t> cand;
    if (!pr.no_candidates)
        for (uint64_t p = lo; p < hi; ++p)
            if (is_candidate(view, pr.T, pr.P, p)) cand.push_back(p);
    return cand;
}

// cdc_exit_kernel, cdc_walk_kernel, cdc_mark_kernel: onchain[i] = 1 for the nodes on the chain from node 0
std::vector<uint8_t> mark_chain(const std::vector<uint32_t>& next) {
    const uint32_t nnodes = (uint32_t)next.size(), nblocks = (nnodes + kNodeBlock - 1) / kNodeBlock;
    auto block_end = [nnodes](uint32_t b) { return b * kNodeBlock + kNodeBlock < nnodes ? b * kNodeBlock + kNodeBlock : nnodes; };
    std::vector<uint32_t> exit_(nnodes), entry(nblocks, kNoEntry);
    for (uint32_t b = 0; b < nblocks; ++b)
        block_exit_seq(next.data() + b * kNodeBlock, b * kNodeBlock, block_end(b), exit_.data() + b * kNodeBlock);
    for (uint32_t cur = 0; cur < nnodes; cur = exit_[cur]) entry[cur / kNodeBlock] = cur;
    std::vector<uint8_t> onchain(nnodes, 0);
    for (uint32_t b = 0; b < nblocks; ++b)
        if (entry[b] != kNoEntry)
            block_mark_seq(next.data() + b * kNodeBlock, b * kNodeBlock, block_end(b), entry[b], onchain.data() + b * kNodeBlock);
    return onchain;
}

struct Selection {
    std::vector<uint64_t> first;   // index of file f's first chunk; first[nfiles] = number of chunks
    uint64_t open_start = 0;       // where the chunk after the last emitted one starts
};

// Cut selection over one layout as ingest.cu's select_cuts / emit_cuts run it: batch_next for every item, the chain, the
// counts of the on-chain nodes and their exclusive scan, batch_first, batch_emit for every on-chain node; out(index,
// offset, size) receives the chunks.  Returns 0, -2 when an item's node is not a fresh one behind it in the chain order
// or -3 when a file's root is off the chain.
template <typename OutT>
int select_cuts(const BatchLayout& B, const CdcParams& P, OutT out, Selection* sel) {
    const uint32_t nnodes = B.ncand + B.nfiles;
    std::vector<uint64_t> npos(nnodes);
    std::vector<uint32_t> next(nnodes, 0), forced(nnodes), cnt(nnodes);
    for (uint32_t i = 0; i < nnodes; ++i) {
        const BatchNext r = batch_next(B, P, i);
        if (r.node >= nnodes || next[r.node] != 0 || r.next <= r.node) return -2;
        npos[r.node] = r.pos;
        next[r.node] = r.next;
        forced[r.node] = r.forced;
        cnt[r.node] = r.count;
    }
    const std::vector<uint8_t> onchain = mark_chain(next);
    std::vector<uint64_t> offsets(nnodes + 1, 0);
    for (uint32_t i = 0; i < nnodes; ++i) offsets[i + 1] = offsets[i] + (onchain[i] ? cnt[i] : 0);
    sel->first.assign(B.nfiles + 1, offsets[nnodes]);
    for (uint32_t f = 0; f < B.nfiles; ++f) {
        const uint32_t root = batch_node_of_root(B, f);
        if (!onchain[root]) return -3;
        sel->first[f] = offsets[root];
    }
    for (uint32_t i = 0; i < nnodes; ++i) {
        if (!onchain[i]) continue;
        const uint64_t base = offsets[i];
        const uint64_t end = batch_emit(B, P, npos[i], forced[i], next[i] < nnodes ? npos[next[i]] : 0ull,
                                        [&](uint64_t k, uint64_t off, uint64_t size) { out(base + k, off, size); });
        if (next[i] == nnodes) sel->open_start = end;
    }
    return 0;
}
}  // namespace

extern "C" {

// Emulates a streaming session fed in slices of `slice` bytes (0 = everything in one feed).
// Returns the number of chunks (may exceed cap), (size_t)-1 on invalid config, (size_t)-2 / -3 on a broken chain.
size_t sim_chunk(const uint8_t* data, size_t n, uint64_t window, uint64_t minc, uint64_t maxc, uint64_t poly,
                 uint64_t mask, int variant, size_t slice, uint64_t* out_offsets, uint64_t* out_sizes, size_t cap) {
    Params pr;
    if (!resolve(window, minc, maxc, poly, mask, variant, &pr)) return (size_t)-1;
    size_t nout = 0;
    uint64_t chunk_start = 0, stream_pos = 0, keep_from = 0;
    if (slice == 0) slice = n ? n : 1;
    for (bool final = false; !final;) {
        size_t len = (size_t)((n - stream_pos) < slice ? (n - stream_pos) : slice);
        final = stream_pos + len == n;
        const uint64_t scan_lo = stream_pos, scan_hi = stream_pos + len;
        // the device sees bytes from keep_from only
        ByteView view{data + keep_from, keep_from, keep_from};
        std::vector<uint64_t> cand = candidates(view, pr, scan_lo, scan_hi);
        // process(): the feed is a layout of one file, from the open chunk's start to scan_hi
        uint64_t dummy = 0;
        BatchLayout B{cand.empty() ? &dummy : cand.data(), (uint32_t)cand.size(), &chunk_start, &scan_hi, 1, final};
        Selection sel;
        int rc = select_cuts(B, pr.P, [&](uint64_t k, uint64_t off, uint64_t size) {
            if (nout + k < cap) {
                out_offsets[nout + k] = off;
                out_sizes[nout + k] = size;
            }
        }, &sel);
        if (rc != 0) return (size_t)rc;
        nout += sel.first[1];
        chunk_start = sel.open_start;   // (the kernel writes scalars[1]; the host reads it after the pass)
        stream_pos = scan_hi;
        uint64_t nk = chunk_start < (stream_pos > (uint64_t)kHistory ? stream_pos - kHistory : 0)
                          ? chunk_start
                          : (stream_pos > (uint64_t)kHistory ? stream_pos - kHistory : 0);
        if (nk < keep_from) nk = keep_from;
        keep_from = nk;
    }
    return nout;
}

// candidate positions through the shared predicate (for direct comparison with the oracle)
size_t sim_candidates(const uint8_t* data, size_t n, uint64_t window, uint64_t poly, uint64_t mask, uint64_t* out,
                      size_t cap) {
    Params pr;
    if (!resolve(window, 1, 2, poly, mask, 0, &pr)) return (size_t)-1;
    ByteView view{data, 0, 0};
    size_t cnt = 0;
    for (uint64_t p = 0; p < n; ++p)
        if (is_candidate(view, pr.T, pr.P, p)) {
            if (cnt < cap) out[cnt] = p;
            ++cnt;
        }
    return cnt;
}

// Emulates chunk_and_hash_batch's device pass (ingest.cu run_batch_group): the files are laid out in one zeroed buffer
// (256-byte aligned starts, >= 64 zero bytes in front of each), ONE candidate pass over the whole buffer, the merged
// node table, the shared chain kernels, per-node emission.  out_first[f] = index of file f's first chunk.
size_t sim_chunk_batch(const uint8_t* const* files, const size_t* lens, size_t nfiles, uint64_t window, uint64_t minc,
                       uint64_t maxc, uint64_t poly, uint64_t mask, int variant, uint64_t* out_offsets, uint64_t* out_sizes,
                       size_t cap, uint64_t* out_first) {
    Params pr;
    if (!resolve(window, minc, maxc, poly, mask, variant, &pr)) return (size_t)-1;
    const uint32_t nf = (uint32_t)nfiles;
    std::vector<uint64_t> starts(nf), ends(nf);
    uint64_t pos = 256;
    for (uint32_t f = 0; f < nf; ++f) {
        starts[f] = pos;
        ends[f] = pos + lens[f];
        pos += (lens[f] + 64 + 255) & ~255ull;
    }
    const uint64_t L = pos;
    std::vector<uint8_t> buf((size_t)L + 256, 0);
    for (uint32_t f = 0; f < nf; ++f)
        if (lens[f]) memcpy(buf.data() + starts[f], files[f], lens[f]);
    std::vector<uint64_t> cand = candidates(ByteView{buf.data(), 0, 0}, pr, 0, L);
    uint64_t dummy = 0;
    BatchLayout B{cand.empty() ? &dummy : cand.data(), (uint32_t)cand.size(), starts.data(), ends.data(), nf, true};
    Selection sel;
    int rc = select_cuts(B, pr.P, [&](uint64_t k, uint64_t off, uint64_t size) {
        if (k < cap) {
            out_offsets[k] = batch_file_offset(B, off);   // batch_rebase_kernel
            out_sizes[k] = size;
        }
    }, &sel);
    if (rc != 0) return (size_t)rc;
    for (uint32_t f = 0; f <= nf; ++f) out_first[f] = sel.first[f];
    return (size_t)sel.first[nf];
}
}
