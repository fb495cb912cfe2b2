// cdc_logic.h -- integer logic of the content-defined chunker, shared by the CUDA kernels
// (cdc.cu) and by a host-side emulation (tests/sim/cdc_sim.cpp) that calls the same functions in
// the same order, so the exact source lines the GPU runs -- candidates, cut selection, chain
// resolution and every chunk's offset and size -- are checked against the oracle on machines
// without a GPU.  No reference code is reproduced here:
// this is the closed-form / data-parallel re-derivation described in DESIGN.md §ingest.
//
// Reference behaviour being matched (paths under /root/reference):
//   table            src/chunking/rabin_fingerprint_table.h:16-26
//   rolling update   src/chunking/rabin_chunker.cpp:80-87, src/chunking/streaming_chunker.cpp:55-68
//   cut rule (S)     include/yams/chunking/streaming_chunker.h:146-181
//   cut rule (R)     src/chunking/rabin_chunker.cpp:63-110
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define YB_HD __host__ __device__ __forceinline__
#else
#define YB_HD inline
#endif

namespace yb {

constexpr uint64_t kDefaultPoly = 0x3DA3358B4DC173ULL;
constexpr int kMaxWindow = 48;   // the reference ring buffer is std::array<std::byte,48>
constexpr int kMaxSteps = 8;     // '<< 8' per byte on a 64-bit state
constexpr int kHistory = kMaxWindow + kMaxSteps;  // bytes of look-behind a position can need

// Resolved chunking parameters (host computes once per call / session).
struct CdcParams {
    uint64_t mask;
    uint64_t lo;       // first testable offset inside a chunk: streaming max(min,1)-1, rabin min
    uint64_t force;    // size of a forced chunk: max(min,max) (streaming: at least 1)
    uint32_t window;   // 1..48
    uint32_t steps;    // rolling steps that can influence the masked bits: 1..8 (0 if mask==0)
    uint32_t nfast;    // number of byte values passing the low-byte prefilter if <= 4, else 0
    uint8_t fast[4];   // those byte values
};

YB_HD uint64_t table_entry(uint64_t poly, uint32_t byte) {
    uint64_t h = 0;
#pragma unroll
    for (int bit = 0; bit < 8; ++bit)
        if (byte & (1u << bit)) h ^= poly << bit;
    return h;
}

YB_HD uint32_t mask_steps(uint64_t mask) {
    if (mask == 0) return 0;
    uint32_t hi = 63;
    while (!((mask >> hi) & 1ull)) --hi;
    return hi / 8 + 1;
}

// Byte reader with stream-start semantics: positions before the stream read as 0 (the reference
// ring is zero-initialised and T[0] == 0).  `data` points at stream position `base_pos`; `lowest`
// is the lowest stream position that is physically readable behind data (history / carry).
struct ByteView {
    const uint8_t* data;   // data[0] is stream position base_pos
    uint64_t base_pos;     // stream position of data[0]
    uint64_t lowest;       // lowest readable stream position (<= base_pos); below it bytes are 0
                           // (only legal when lowest == 0, i.e. the true stream start)
    YB_HD uint32_t at(int64_t pos) const {
        if (pos < (int64_t)lowest) return 0;
        return data[pos - (int64_t)base_pos];
    }
};

// Masked rolling-hash value at stream position p, rebuilt from `steps` local bytes.  Bits below
// 8*steps equal the reference's full 64-bit state because '<<8' and '-' only carry information
// upward.  T is the 256-entry table (shared/constant memory on device).
template <typename ViewT, typename TableT>
YB_HD bool is_candidate(const ViewT& v, const TableT& T, const CdcParams& P, uint64_t p) {
    uint64_t h = 0;
    for (int j = (int)P.steps - 1; j >= 0; --j) {
        int64_t q = (int64_t)p - j;
        if (q < 0) continue;  // before the stream start the state is still 0
        uint32_t nb = v.at(q);
        uint32_t ob = v.at(q - (int64_t)P.window);
        h = ((h - T[ob]) << 8) ^ T[nb];
    }
    return (h & P.mask) == P.mask;
}

// ---- cut selection --------------------------------------------------------------------------
// cand[0..ncand) ascending stream positions of candidates (only those >= the session's first
// scanned position are present; earlier ones are provably irrelevant, see DESIGN.md).
// From a chunk starting at `s`, find the next cut that lands on a candidate.
//   returns index j of that candidate (cut after byte cand[j]) and the number F of forced
//   (max-size) chunks emitted before it; j == ncand means "no further candidate cut" (END).
struct NextCut {
    uint32_t j;
    uint64_t forced;
};

YB_HD uint32_t lower_bound_u64(const uint64_t* a, uint32_t lo, uint32_t hi, uint64_t key) {
    // first index in [lo,hi) with a[idx] >= key
    while (lo < hi) {
        uint32_t mid = lo + ((hi - lo) >> 1);
        if (a[mid] < key) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// galloping search from a hint (candidates are ~1/8192 dense, the answer is usually 1-3 ahead)
YB_HD uint32_t gallop_lower_bound(const uint64_t* a, uint32_t from, uint32_t n, uint64_t key) {
    if (from >= n || a[from] >= key) return from;
    uint32_t step = 1, lo = from, hi = from + 1;
    while (hi < n && a[hi] < key) {
        lo = hi;
        step <<= 1;
        hi = (hi + step < n) ? hi + step : n;
    }
    return lower_bound_u64(a, lo + 1, hi, key);
}

YB_HD NextCut next_cut(const uint64_t* cand, uint32_t ncand, uint32_t hint, uint64_t s,
                       const CdcParams& P) {
    NextCut r;
    uint64_t t = 0;
    uint32_t j = hint;
    for (;;) {
        uint64_t st = s + t * P.force;
        j = gallop_lower_bound(cand, j, ncand, st + P.lo);
        if (j >= ncand) { r.j = ncand; r.forced = 0; return r; }
        uint64_t c = cand[j];
        uint64_t t2 = (c - s) / P.force;
        uint64_t st2 = s + t2 * P.force;
        if (c - st2 >= P.lo) { r.j = j; r.forced = t2; return r; }
        t = t2;  // c sits in the untested head of forced chunk t2: keep looking inside that chunk
        // next probe key is st2 + lo > c, so j strictly advances
    }
}


// ---- chain resolution over "nodes" ------------------------------------------------------------
// The nodes of a layout (below) are the chunk starts it can have, numbered by position.  next[node] is the node of the next
// cut, or END = nnodes.  next[node] > node always, so a block of consecutive nodes can be resolved by a single backward pass.
constexpr uint32_t kNodeBlock = 1024;
constexpr uint32_t kNoEntry = 0xFFFFFFFFu;

// exit_out[i] = first node >= blk_end reached from node blk_start+i by following next[]
YB_HD void block_exit_seq(const uint32_t* next_blk, uint32_t blk_start, uint32_t blk_end,
                          uint32_t* exit_blk) {
    for (uint32_t i = blk_end; i-- > blk_start;) {
        uint32_t nx = next_blk[i - blk_start];
        exit_blk[i - blk_start] = nx >= blk_end ? nx : exit_blk[nx - blk_start];
    }
}

// mark every node of [blk_start, blk_end) that lies on the chain entered at `entry`
YB_HD void block_mark_seq(const uint32_t* next_blk, uint32_t blk_start, uint32_t blk_end,
                          uint32_t entry, uint8_t* onchain_blk) {
    uint32_t cur = entry;
    while (cur < blk_end) {
        onchain_blk[cur - blk_start] = 1;
        cur = next_blk[cur - blk_start];
    }
}

// ---- cut selection over a layout of files ----------------------------------------------------------------------------
// File f occupies positions [starts[f], ends[f]).  chunk_and_hash_batch lays many files out in one buffer (ascending, zero
// gaps of >= 64 bytes in front of every file); a streaming feed is a layout of one file that starts at the open chunk and
// ends at the last fed byte, final when the stream ends there.
// Nodes = file roots + candidate cuts merged by position (a root sorts before a candidate at the same position).  The chain
// runs root(0) -> cuts of file 0 -> root(1) -> ...; nodes lying in a gap or at a file's end are dead links.
struct BatchLayout {
    const uint64_t* cand;     // ascending candidate positions of the whole buffer
    uint32_t ncand;
    const uint64_t* starts;
    const uint64_t* ends;
    uint32_t nfiles;
    bool final;               // the last file is complete; otherwise the stream goes on past ends[nfiles - 1]
};
constexpr uint32_t kBatchTail = 0x80000000u;       // forced[]: the node's chunks run to the end of its file

YB_HD uint32_t upper_bound_u64(const uint64_t* a, uint32_t n, uint64_t key) {   // first idx with a[idx] > key
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        uint32_t mid = lo + ((hi - lo) >> 1);
        if (a[mid] <= key) lo = mid + 1; else hi = mid;
    }
    return lo;
}
// node index of candidate j (the chunk that starts at cand[j] + 1)
YB_HD uint32_t batch_node_of_cand(const BatchLayout& B, uint32_t j) { return j + upper_bound_u64(B.starts, B.nfiles, B.cand[j] + 1); }
// node index of the root of file f
YB_HD uint32_t batch_node_of_root(const BatchLayout& B, uint32_t f) {
    uint64_t s = B.starts[f];
    return f + (s == 0 ? 0u : lower_bound_u64(B.cand, 0, B.ncand, s - 1));   // candidates with cand + 1 < s
}
// offset of layout position pos inside the file that holds it
YB_HD uint64_t batch_file_offset(const BatchLayout& B, uint64_t pos) { return pos - B.starts[upper_bound_u64(B.starts, B.nfiles, pos) - 1]; }
// Chunks of the tail [s, ends[f]) of file f: all of it, the remainder included (streaming_chunker.h:115-118,
// rabin_chunker.cpp:66-67 min(start+max, size)), unless the stream goes on past the file: then the remainder stays open.
YB_HD uint64_t batch_tail_count(const BatchLayout& B, uint32_t f, uint64_t s, uint64_t force) {
    const uint64_t rem = B.ends[f] - s;
    return (B.final || f + 1 < B.nfiles) ? (rem + force - 1) / force : rem / force;
}
struct BatchNext {
    uint32_t node;     // node index of the item
    uint64_t pos;      // start position of the node
    uint32_t next;     // node index, nnodes = END
    uint32_t forced;   // forced chunks before the candidate cut, or kBatchTail
    uint32_t count;    // chunks this node emits when it is on the chain
};
// Selection step of item i: candidate i (i < ncand) or the root of file i - ncand.
YB_HD BatchNext batch_next(const BatchLayout& B, const CdcParams& P, uint32_t i) {
    BatchNext r;
    uint32_t hint;
    if (i < B.ncand) {
        r.pos = B.cand[i] + 1;   // a cut after byte cand[i] starts the next chunk at cand[i] + 1
        r.node = batch_node_of_cand(B, i);
        hint = i + 1;
    } else {
        const uint32_t f = i - B.ncand;
        r.pos = B.starts[f];
        r.node = batch_node_of_root(B, f);
        hint = lower_bound_u64(B.cand, 0, B.ncand, r.pos);
    }
    r.next = r.node + 1;
    r.forced = 0;
    r.count = 0;
    const uint32_t fup = upper_bound_u64(B.starts, B.nfiles, r.pos);   // files starting at or before pos
    if (fup == 0 || r.pos >= B.ends[fup - 1]) return r;                // gap / file end: dead link
    const uint32_t f = fup - 1;
    NextCut c = next_cut(B.cand, B.ncand, hint, r.pos, P);
    if (c.j < B.ncand && B.cand[c.j] < B.ends[f]) {
        r.next = batch_node_of_cand(B, c.j);
        r.forced = (uint32_t)c.forced;
        r.count = r.forced + 1;
    } else {
        r.next = f + 1 < B.nfiles ? batch_node_of_root(B, f + 1) : B.ncand + B.nfiles;
        r.forced = kBatchTail;
        r.count = (uint32_t)batch_tail_count(B, f, r.pos, P.force);
    }
    return r;
}
// Chunks of an on-chain node that starts at s: emit(k, offset, size) for k = 0 .. count-1.  next_pos = start position of
// next[node].  Returns the position after the node's chunks, which for the last node of the chain is the new open-chunk start.
template <typename EmitT>
YB_HD uint64_t batch_emit(const BatchLayout& B, const CdcParams& P, uint64_t s, uint32_t forced, uint64_t next_pos, EmitT emit) {
    const uint32_t fup = upper_bound_u64(B.starts, B.nfiles, s);
    if (fup == 0 || s >= B.ends[fup - 1]) return s;   // dead link
    if (forced & kBatchTail) {
        const uint64_t e = B.ends[fup - 1];
        const uint64_t n = batch_tail_count(B, fup - 1, s, P.force);
        for (uint64_t t = 0; t < n; ++t) {
            uint64_t cs = s + t * P.force;
            emit(t, cs, e - cs < P.force ? e - cs : P.force);
        }
        const uint64_t ns = s + n * P.force;
        return ns < e ? ns : e;
    }
    for (uint32_t t = 0; t < forced; ++t) emit((uint64_t)t, s + (uint64_t)t * P.force, P.force);
    const uint64_t ls = s + (uint64_t)forced * P.force;
    emit((uint64_t)forced, ls, next_pos - ls);
    return next_pos;
}

}  // namespace yb
