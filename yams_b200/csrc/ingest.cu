// ingest.cu -- host orchestration of the content-ingest path: CDC boundaries + per-chunk SHA-256.
// Implements the content_ingest_v1 entry points of include/yams_b200.h.
//
// Reference call sites this replaces (paths under /root/reference):
//   StreamingChunker::chunkData       src/chunking/streaming_chunker.cpp:92-137
//   StreamingChunker::processStream   include/yams/chunking/streaming_chunker.h:78-121
//   RabinChunker::chunkDataImpl       src/chunking/rabin_chunker.cpp:120-152
//   ContentStore::store / storeBytes  src/api/content_store_impl.cpp:216-220, 510-545 (callers)
#include <stdlib.h>

#include <algorithm>
#include <chrono>
#include <memory>
#include <mutex>
#include <thread>
#include <new>
#include <vector>

#include "cdc_kernels.cuh"
#include "upload.cuh"

namespace yb {

constexpr uint32_t kTileBytesHost = kTileBytes;
// Device-resident data is processed in segments (two host round trips each to size the selection buffers).  16 GiB segments
// keep those round trips rare; the candidate workspace grows to ~1 GiB (2 x 16 B per 4 KiB tile x 16-entry slack).
static uint64_t segment_bytes() {
    const char* e = getenv("YAMS_B200_SEGMENT_MIB");
    uint64_t mib = e ? strtoull(e, nullptr, 10) : 16384;
    if (mib < 1) mib = 1;
    if (mib > 16384) mib = 16384;
    return mib << 20;
}
static inline double now_ms() {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
}
constexpr uint64_t kFeedSlice = 256ull << 20;      // host feeds are staged 256 MiB at a time

// All device-side resources of one ingest stream: the chunking and hashing workspace, the two staging buffers of the host
// path and the pinned images of the upload path.  They are pooled: `yams add` calls chunk_and_hash once per file, and
// cudaMalloc / cudaFree of the workspace would otherwise dominate small inputs.
struct IngestRes {
    DeviceCtx* dev = nullptr;
    cudaStream_t st = nullptr;       // kernels
    cudaStream_t copy_st = nullptr;  // H2D copies of the streaming session
    CdcParams P{};
    bool no_candidates = false;  // lo >= force: no candidate can ever cut
    DevBuf table, tile_counts, tile_offsets, cand, cand_tmp, next, forced, exit_, entry, onchain, emit_counts,
        emit_offsets, scan_scratch, descs, scalars, sha_order;
    DevBuf npos, fileinfo, first;   // node start positions, file layout [starts | ends], per-file chunk ranges (batch)
    DevBuf stage[2];             // device copies of host input
    HostBuf h_scalars;           // pinned: [0] ncand/ntotal, [1] new chunk start, [6..7] layout of a feed
    HostBuf pin[2];              // pinned images of two device-buffer slices (staged_upload)
    uint64_t ndescs = 0;         // chunks accumulated in `descs`
    uint64_t chunk_start = 0;    // stream position where the open chunk starts
    cudaEvent_t ev[4] = {};      // stage marks of one process(), one batch group or one session hash
    cudaEvent_t call[3] = {};    // whole-call marks: start, chunking done, hashing done
    cudaEvent_t copied[2] = {};  // session: H2D copy into stage[b] finished
    cudaEvent_t freed[2] = {};   // session: stage[b] no longer read
    cudaEvent_t pin_done[2] = {};  // H2D copy out of pin[b] finished
    float ms_scan = 0, ms_select = 0;
    double host_sync1 = 0, host_sync2 = 0, host_alloc = 0, host_total = 0;  // wall-clock ms (diagnostics)

    bool created = false;
    yams_status_t create() {
        if (created) return YAMS_OK;
        yams_status_t rc = ensure_device(&dev);
        if (rc != YAMS_OK) return rc;
        YB_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
        YB_CUDA(cudaStreamCreateWithFlags(&copy_st, cudaStreamNonBlocking));
        for (cudaEvent_t* e : {&ev[0], &ev[1], &ev[2], &ev[3], &call[0], &call[1], &call[2]}) YB_CUDA(cudaEventCreate(e));
        for (cudaEvent_t* e : {&copied[0], &copied[1], &freed[0], &freed[1], &pin_done[0], &pin_done[1]})
            YB_CUDA(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
        if ((rc = table.reserve(256 * 8)) != YAMS_OK) return rc;
        if ((rc = scalars.reserve(64)) != YAMS_OK) return rc;
        if ((rc = h_scalars.reserve(64 + 256 * 8)) != YAMS_OK) return rc;
        created = true;
        return YAMS_OK;
    }
    // (re)configure for a new stream: parameters, table, counters. Buffers are kept.
    yams_status_t init(const yams_cdc_config* cfg) {
        uint64_t* tbl = h_scalars.as<uint64_t>() + 8;   // pinned staging for the table
        YB_CUDA(cudaStreamSynchronize(st));
        yams_status_t rc = resolve_params(cfg, &P, tbl);
        if (rc != YAMS_OK) return rc;
        no_candidates = P.lo >= P.force;
        ndescs = 0;
        chunk_start = 0;
        ms_scan = ms_select = 0;
        host_sync1 = host_sync2 = host_alloc = host_total = 0;
        YB_CUDA(cudaMemcpyAsync(table.p, tbl, 256 * 8, cudaMemcpyHostToDevice, st));
        return YAMS_OK;
    }
    // both streams are drained first, so the buffers may be freed in any order after they are destroyed
    ~IngestRes() {
        if (st) cudaStreamSynchronize(st);
        if (copy_st) cudaStreamSynchronize(copy_st);
        for (cudaEvent_t e : {ev[0], ev[1], ev[2], ev[3], call[0], call[1], call[2], copied[0], copied[1], freed[0], freed[1],
                              pin_done[0], pin_done[1]})
            if (e) cudaEventDestroy(e);
        for (cudaStream_t s : {st, copy_st})
            if (s) cudaStreamDestroy(s);
    }

    // Waits for the kernel stream; the host time spent waiting is added to *acc.
    yams_status_t wait(double* acc) {
        const double t0 = now_ms();
        YB_CUDA(cudaStreamSynchronize(st));
        *acc += now_ms() - t0;
        return YAMS_OK;
    }

    // Candidate scan of stream positions [scan_lo, scan_hi): the ascending candidate positions land in `cand`,
    // their number in *ncand_out.  Single pass; dense (adversarial) data falls back to the exact two-pass kernels.
    yams_status_t scan(const uint8_t* data, uint64_t base_pos, uint64_t lowest, uint64_t scan_lo, uint64_t scan_hi,
                       uint32_t* ncand_out) {
        yams_status_t rc;
        uint64_t* d_sc = scalars.as<uint64_t>();
        volatile uint64_t* h_sc = h_scalars.as<uint64_t>();
        uint32_t ncand = 0;
        if (!cand.p && (rc = cand.reserve(8)) != YAMS_OK) return rc;   // a valid pointer even when there is no candidate
        if (!no_candidates && scan_hi > scan_lo) {
            // tiles start at a 16-byte-aligned ADDRESS: normally at or below scan_lo (the positions in
            // [origin, scan_lo) are masked and never dereferenced); when that would fall before stream position
            // 0 (misaligned buffer at the very start of a stream) the tiles start at the next aligned address
            // and the < 16 head positions [scan_lo, origin) are tested separately by the kernels.
            uintptr_t addr_lo = reinterpret_cast<uintptr_t>(data) + (scan_lo - base_pos);
            uint64_t mis = (uint64_t)(addr_lo & 15);
            uint64_t origin = scan_lo >= mis ? scan_lo - mis : scan_lo + (16 - mis);
            uint64_t span = scan_hi > origin ? scan_hi - origin : 1;
            uint64_t ntiles64 = (span + kTileBytesHost - 1) / kTileBytesHost;
            YB_ARG(ntiles64 < (1ull << 31), "segment too large");
            uint32_t ntiles = (uint32_t)ntiles64;
            ScanArgs A{data, base_pos, lowest, origin, scan_lo, scan_hi, table.as<uint64_t>(), P};
            // single pass: every warp scans a contiguous range (4 KiB tiles) and appends to its own slice
            uint32_t ntiles4 = (uint32_t)((span + kSinglePassTile - 1) / kSinglePassTile);
            uint32_t nslices = std::min<uint32_t>(ntiles4, (uint32_t)dev->sm_count * kSinglePassWarpsPerCta);
            uint32_t tpw = (ntiles4 + nslices - 1) / nslices;
            uint32_t slice_cap = std::max<uint32_t>(64u, tpw * 16u);   // 32x the 1/8192 density of random data
            size_t total_cap = (size_t)nslices * slice_cap;
            if ((rc = cand_tmp.reserve(total_cap * 8)) != YAMS_OK) return rc;
            if ((rc = cand.reserve(total_cap * 8)) != YAMS_OK) return rc;
            if ((rc = tile_counts.reserve((size_t)std::max<uint32_t>(ntiles, nslices) * 4)) != YAMS_OK) return rc;
            if ((rc = launch_scan_single_pass(A, ntiles4, cand_tmp.as<uint64_t>(), tile_counts.as<uint32_t>(), slice_cap,
                                              nslices, cand.as<uint64_t>(), d_sc, st)) != YAMS_OK)
                return rc;
            YB_CUDA(cudaMemcpyAsync((void*)h_sc, d_sc, 24, cudaMemcpyDeviceToHost, st));
            if ((rc = wait(&host_sync1)) != YAMS_OK) return rc;
            if (h_sc[2] == 0) {
                YB_ARG(h_sc[0] < 0xFFFFFFF0ull, "too many boundary candidates in one segment");
                ncand = (uint32_t)h_sc[0];
            } else {
                // dense candidates overflowed a slice: the exact two-pass kernels take over
                if ((rc = tile_counts.reserve((size_t)ntiles * 4)) != YAMS_OK) return rc;
                if ((rc = tile_offsets.reserve((size_t)ntiles * 4)) != YAMS_OK) return rc;
                uint32_t grid = std::min<uint32_t>(ntiles, (uint32_t)dev->sm_count * 8u);
                cdc_count_kernel<<<grid, 256, 0, st>>>(A, ntiles, tile_counts.as<uint32_t>());
                if ((rc = exclusive_scan_u32(tile_counts.as<uint32_t>(), tile_offsets.as<uint32_t>(), ntiles,
                                             d_sc + 0, scan_scratch, st)) != YAMS_OK)
                    return rc;
                YB_CUDA(cudaMemcpyAsync((void*)h_sc, d_sc, 8, cudaMemcpyDeviceToHost, st));
                if ((rc = wait(&host_sync1)) != YAMS_OK) return rc;
                uint64_t nc = h_sc[0];
                YB_ARG(nc < 0xFFFFFFF0ull, "too many boundary candidates in one segment");
                ncand = (uint32_t)nc;
                if (ncand) {
                    if ((rc = cand.reserve((size_t)ncand * 8)) != YAMS_OK) return rc;
                    cdc_write_kernel<<<grid, 256, 0, st>>>(A, ntiles, tile_counts.as<uint32_t>(),
                                                           tile_offsets.as<uint32_t>(), cand.as<uint64_t>());
                }
            }
        }
        *ncand_out = ncand;
        return YAMS_OK;
    }

    // ---- cut selection over a layout (cdc_logic.h): one streaming feed, or the files of a batch group ----
    yams_status_t reserve_nodes(uint32_t nnodes) {
        const uint32_t nblocks = (nnodes + kNodeBlock - 1) / kNodeBlock;
        yams_status_t rc;
        if ((rc = npos.reserve((size_t)nnodes * 8)) != YAMS_OK) return rc;
        for (DevBuf* b : {&next, &forced, &exit_})
            if ((rc = b->reserve((size_t)nnodes * 4)) != YAMS_OK) return rc;
        if ((rc = entry.reserve((size_t)nblocks * 4)) != YAMS_OK) return rc;
        if ((rc = onchain.reserve((size_t)nnodes)) != YAMS_OK) return rc;
        for (DevBuf* b : {&emit_counts, &emit_offsets})
            if ((rc = b->reserve((size_t)nnodes * 4)) != YAMS_OK) return rc;
        return YAMS_OK;
    }
    // onchain[i] = 1 for the nodes on the chain of cuts that starts at node 0; every byte of onchain[0, nnodes) is written
    yams_status_t mark_chain(uint32_t nnodes) {
        const uint32_t nblocks = (nnodes + kNodeBlock - 1) / kNodeBlock;
        cdc_exit_kernel<<<nblocks, 32, 0, st>>>(next.as<uint32_t>(), nnodes, exit_.as<uint32_t>());
        YB_CUDA(cudaMemsetAsync(entry.p, 0xFF, (size_t)nblocks * 4, st));
        cdc_walk_kernel<<<1, 32, 0, st>>>(exit_.as<uint32_t>(), nnodes, entry.as<uint32_t>());
        cdc_mark_kernel<<<nblocks, 32, 0, st>>>(next.as<uint32_t>(), nnodes, entry.as<uint32_t>(), onchain.as<uint8_t>());
        return YAMS_OK;
    }
    // emit_offsets = exclusive scan of emit_counts; *total (their sum) is read back to the host
    yams_status_t count_offsets(uint32_t nnodes, uint64_t* total) {
        uint64_t* d_sc = scalars.as<uint64_t>();
        yams_status_t rc = exclusive_scan_u32(emit_counts.as<uint32_t>(), emit_offsets.as<uint32_t>(), nnodes, d_sc + 0,
                                              scan_scratch, st);
        if (rc != YAMS_OK) return rc;
        YB_CUDA(cudaMemcpyAsync(h_scalars.p, d_sc, 8, cudaMemcpyDeviceToHost, st));
        if ((rc = wait(&host_sync2)) != YAMS_OK) return rc;
        *total = h_scalars.as<volatile uint64_t>()[0];
        return YAMS_OK;
    }
    // The next cut from every node, the chain from node 0, the chunk counts of its nodes and their offsets; *total is the
    // number of chunks emit_cuts writes.
    yams_status_t select_cuts(const BatchArgs& B, uint64_t* total) {
        const uint32_t nnodes = B.L.ncand + B.L.nfiles;
        yams_status_t rc = reserve_nodes(nnodes);
        if (rc != YAMS_OK) return rc;
        const uint32_t tgrid = (nnodes + 255) / 256;
        batch_next_kernel<<<tgrid, 256, 0, st>>>(B, npos.as<uint64_t>(), next.as<uint32_t>(), forced.as<uint32_t>(),
                                                 emit_counts.as<uint32_t>());
        if ((rc = mark_chain(nnodes)) != YAMS_OK) return rc;
        batch_mask_counts_kernel<<<tgrid, 256, 0, st>>>(onchain.as<uint8_t>(), emit_counts.as<uint32_t>(), nnodes);
        return count_offsets(nnodes, total);
    }
    // The selected chunks to out[0, total), the open-chunk start to scalars[1].
    yams_status_t emit_cuts(const BatchArgs& B, yams_chunk_desc* out) {
        const uint32_t nnodes = B.L.ncand + B.L.nfiles;
        batch_emit_kernel<<<(nnodes + 255) / 256, 256, 0, st>>>(B, npos.as<uint64_t>(), next.as<uint32_t>(), forced.as<uint32_t>(),
                                                                onchain.as<uint8_t>(), emit_offsets.as<uint32_t>(), out,
                                                                scalars.as<uint64_t>() + 1);
        YB_CUDA(cudaGetLastError());
        return YAMS_OK;
    }

    // Scan stream positions [scan_lo, scan_hi) (bytes readable from `lowest`), select cuts from the
    // open chunk at chunk_start, append the completed chunks to descs. `data[0]` is stream position
    // base_pos.  When final, the trailing partial chunk is emitted too.
    yams_status_t process(const uint8_t* data, uint64_t base_pos, uint64_t lowest, uint64_t scan_lo,
                          uint64_t scan_hi, bool final) {
        yams_status_t rc;
        const double t_begin = now_ms();
        uint64_t* d_sc = scalars.as<uint64_t>();
        volatile uint64_t* h_sc = h_scalars.as<uint64_t>();
        uint32_t ncand = 0;
        YB_CUDA(cudaEventRecord(ev[0], st));
        // The feed is a layout of one file, from the open chunk's start to scan_hi.  Its upload is queued ahead of the scan,
        // so that it is not on the path from the host's wait for the scan to the selection kernels.
        uint64_t* lay = h_scalars.as<uint64_t>() + 6;   // pinned; the copy out of it ended with the previous process()
        lay[0] = chunk_start;
        lay[1] = scan_hi;
        if ((rc = fileinfo.reserve(16)) != YAMS_OK) return rc;
        YB_CUDA(cudaMemcpyAsync(fileinfo.p, lay, 16, cudaMemcpyHostToDevice, st));
        if ((rc = scan(data, base_pos, lowest, scan_lo, scan_hi, &ncand)) != YAMS_OK) return rc;
        YB_CUDA(cudaEventRecord(ev[1], st));
        const BatchArgs B{BatchLayout{cand.as<uint64_t>(), ncand, fileinfo.as<uint64_t>(), fileinfo.as<uint64_t>() + 1, 1, final}, P};
        uint64_t nnew = 0;
        if ((rc = select_cuts(B, &nnew)) != YAMS_OK) return rc;
        { const double t0 = now_ms();
          if ((rc = descs.reserve((size_t)(ndescs + nnew + 1) * sizeof(yams_chunk_desc), true, st)) != YAMS_OK)
            return rc;
          host_alloc += now_ms() - t0; }
        if ((rc = emit_cuts(B, descs.as<yams_chunk_desc>() + ndescs)) != YAMS_OK) return rc;
        YB_CUDA(cudaMemcpyAsync((void*)(h_sc + 1), d_sc + 1, 8, cudaMemcpyDeviceToHost, st));
        YB_CUDA(cudaEventRecord(ev[2], st));
        YB_CUDA(cudaStreamSynchronize(st));
        chunk_start = h_sc[1];
        ndescs += nnew;
        float a = 0, b = 0;
        cudaEventElapsedTime(&a, ev[0], ev[1]);
        cudaEventElapsedTime(&b, ev[1], ev[2]);
        ms_scan += a;
        ms_select += b;
        host_total += now_ms() - t_begin;
        return YAMS_OK;
    }

    // SHA-256 of descs[first, first + n) over `data` (data[0] is stream position base_pos); total_bytes / n is the mean
    // chunk size the longest-first order buckets by.
    yams_status_t hash(const uint8_t* data, uint64_t base_pos, uint64_t first, uint64_t n, uint64_t total_bytes) {
        if (n == 0) return YAMS_OK;
        if (n >= 0xFFFFFFFFull) {
            set_last_error("too many chunks");
            return YAMS_ERR_INVALID_ARG;
        }
        yams_status_t rc = sha_order.reserve(sha256_order_ws_bytes(n));
        if (rc != YAMS_OK) return rc;
        return launch_sha256_chunks(data, base_pos, descs.as<yams_chunk_desc>(), (uint32_t)first, (uint32_t)n,
                                    reinterpret_cast<unsigned int*>(scalars.as<uint64_t>() + 4), dev->sm_count, st,
                                    sha_order.as<uint32_t>(), total_bytes);
    }
    // Digests of the host table h (offset / size into d_data) into digests[32 * i], through descs.
    yams_status_t hash_table(const uint8_t* d_data, std::vector<yams_chunk_desc>& h, uint64_t total_bytes, uint8_t* digests) {
        const size_t n = h.size();
        yams_status_t rc = descs.reserve(n * sizeof(yams_chunk_desc));
        if (rc != YAMS_OK) return rc;
        YB_CUDA(cudaMemcpyAsync(descs.p, h.data(), n * sizeof(yams_chunk_desc), cudaMemcpyHostToDevice, st));
        if ((rc = hash(d_data, 0, 0, n, total_bytes)) != YAMS_OK) return rc;
        YB_CUDA(cudaMemcpyAsync(h.data(), descs.p, n * sizeof(yams_chunk_desc), cudaMemcpyDeviceToHost, st));
        YB_CUDA(cudaStreamSynchronize(st));
        for (size_t i = 0; i < n; ++i) memcpy(digests + 32 * i, h[i].digest, 32);
        return YAMS_OK;
    }

    // size the descriptor table of a len-byte stream once: every chunk but the last is at least max(min_chunk,1) bytes long
    yams_status_t presize_descs(uint64_t len) {
        const uint64_t per = std::max<uint64_t>(P.lo + 1, 4096);
        return descs.reserve((size_t)(len / per + 16) * sizeof(yams_chunk_desc));
    }
};

static thread_local float g_last_ms[8] = {0};

// The one writer of the ingest_last_timings slots: [0..3] device ms of the candidate scan, the cut selection, SHA-256 and
// the whole call; [4..7] the host ms that r spent in its two waits, in descriptor-table growth and in process() (0 without r).
static void report_timings(const float (&dev_ms)[4], const IngestRes* r) {
    for (int i = 0; i < 4; ++i) g_last_ms[i] = dev_ms[i];
    g_last_ms[4] = r ? (float)r->host_sync1 : 0.f;
    g_last_ms[5] = r ? (float)r->host_sync2 : 0.f;
    g_last_ms[6] = r ? (float)r->host_alloc : 0.f;
    g_last_ms[7] = r ? (float)r->host_total : 0.f;
}

static std::mutex g_pool_mu;
static std::vector<IngestRes*> g_pool;
// one parked resource set per concurrently ingesting host thread (`yams add` workers); creating/destroying one costs
// cudaMalloc/cudaFree/cudaMallocHost calls that serialise the whole device
static size_t pool_max() {
    static const size_t v = [] { const char* e = getenv("YAMS_B200_POOL_MAX"); long x = e ? atol(e) : 16; return (size_t)(x < 1 ? 1 : x); }();
    return v;
}

// cfg == nullptr: the caller only hashes, so no chunking parameters are loaded
static yams_status_t acquire_res(const yams_cdc_config* cfg, IngestRes** out) {
    IngestRes* r = nullptr;
    {
        // a pooled resource may be picked up by a thread that never touched CUDA: bind the plugin's device first
        DeviceCtx* dev = nullptr;
        yams_status_t drc = ensure_device(&dev);
        if (drc != YAMS_OK) return drc;
    }
    {
        std::lock_guard<std::mutex> lk(g_pool_mu);
        if (!g_pool.empty()) {
            r = g_pool.back();
            g_pool.pop_back();
        }
    }
    if (!r) r = new (std::nothrow) IngestRes();
    if (!r) return YAMS_ERR_INTERNAL;
    yams_status_t rc = r->create();
    if (rc == YAMS_OK) rc = cfg ? r->init(cfg) : YAMS_OK;
    if (rc != YAMS_OK) {
        delete r;
        return rc;
    }
    *out = r;
    return YAMS_OK;
}

static void release_res(IngestRes* r) {
    if (!r) return;
    if (r->st) cudaStreamSynchronize(r->st);
    if (r->copy_st) cudaStreamSynchronize(r->copy_st);
    // drop very large buffers instead of parking them in the pool
    const size_t kKeep = 1ull << 30;
    for (DevBuf* b : {&r->stage[0], &r->stage[1], &r->descs, &r->cand, &r->cand_tmp})
        if (b->cap > kKeep) b->release();
    {
        std::lock_guard<std::mutex> lk(g_pool_mu);
        if (g_pool.size() < pool_max()) {
            g_pool.push_back(r);
            return;
        }
    }
    delete r;
}

// A pooled workspace held for the lifetime of the lease; rc says whether one could be had (r is null otherwise).
struct IngestLease {
    IngestRes* r = nullptr;
    yams_status_t rc;
    explicit IngestLease(const yams_cdc_config* cfg) : rc(acquire_res(cfg, &r)) {}
    ~IngestLease() { release_res(r); }
    IngestLease(const IngestLease&) = delete;
    IngestLease& operator=(const IngestLease&) = delete;
};

static yams_status_t copy_out(IngestRes& r, uint64_t first, uint64_t n, yams_chunk_desc** out, size_t* out_n) {
    *out = nullptr;
    *out_n = 0;
    if (n == 0) return YAMS_OK;
    yams_chunk_desc* h = static_cast<yams_chunk_desc*>(malloc((size_t)n * sizeof(yams_chunk_desc)));
    if (!h) {
        set_last_error("out of host memory for %llu chunk descriptors", (unsigned long long)n);
        return YAMS_ERR_INTERNAL;
    }
    cudaError_t e = cudaMemcpyAsync(h, r.descs.as<yams_chunk_desc>() + first, (size_t)n * sizeof(yams_chunk_desc),
                                    cudaMemcpyDeviceToHost, r.st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(r.st);
    if (e != cudaSuccess) {
        free(h);
        set_last_error("D2H of chunk descriptors failed: %s", cudaGetErrorString(e));
        return YAMS_ERR_INTERNAL;
    }
    *out = h;
    *out_n = (size_t)n;
    return YAMS_OK;
}

// One-shot over device-resident data.
static yams_status_t run_device(const uint8_t* d_data, size_t len, const yams_cdc_config* cfg, yams_chunk_desc** out,
                                size_t* out_n) {
    IngestLease ws(cfg);
    if (ws.rc != YAMS_OK) return ws.rc;
    IngestRes& r = *ws.r;
    yams_status_t rc = r.presize_descs(len);
    if (rc != YAMS_OK) return rc;
    YB_CUDA(cudaEventRecord(r.call[0], r.st));
    const uint64_t seg = segment_bytes();
    for (uint64_t lo = 0; lo < len; lo += seg) {
        uint64_t hi = std::min<uint64_t>(len, lo + seg);
        if ((rc = r.process(d_data, 0, 0, lo, hi, hi == len)) != YAMS_OK) return rc;
    }
    YB_CUDA(cudaEventRecord(r.call[1], r.st));
    if ((rc = r.hash(d_data, 0, 0, r.ndescs, len)) != YAMS_OK) return rc;
    YB_CUDA(cudaEventRecord(r.call[2], r.st));
    if ((rc = copy_out(r, 0, r.ndescs, out, out_n)) != YAMS_OK) return rc;
    float t_sha = 0, t_all = 0;
    cudaEventElapsedTime(&t_sha, r.call[1], r.call[2]);
    cudaEventElapsedTime(&t_all, r.call[0], r.call[2]);
    report_timings({r.ms_scan, r.ms_select, t_sha, t_all}, &r);
    return YAMS_OK;
}

// Writes the image of layout positions [lo, hi) to dst: the bytes of the pieces (ascending, disjoint), zeros elsewhere.
static void layout_image(const std::vector<LayoutPiece>& pieces, uint8_t* dst, uint64_t lo, uint64_t hi) {
    // first piece that ends beyond lo
    size_t j = std::partition_point(pieces.begin(), pieces.end(), [lo](const LayoutPiece& x) { return x.pos + x.len <= lo; }) -
               pieces.begin();
    uint64_t p = lo;
    for (; j < pieces.size() && p < hi; ++j) {
        const LayoutPiece& x = pieces[j];
        if (x.pos > p) {   // gap before the piece
            const uint64_t e = std::min<uint64_t>(hi, x.pos);
            memset(dst + (p - lo), 0, (size_t)(e - p));
            p = e;
        }
        const uint64_t e = std::min<uint64_t>(hi, x.pos + x.len);
        if (e > p) {
            memcpy(dst + (p - lo), x.src + (p - x.pos), (size_t)(e - p));
            p = e;
        }
    }
    if (p < hi) memset(dst + (p - lo), 0, (size_t)(hi - p));
}

// Upload of a packed layout (layout_image) whose pieces sit in ordinary (pageable) host memory.  A plain cudaMemcpy moves
// pageable memory at ~10 GB/s through the driver's single staging thread; here host threads assemble each slice of the
// destination in one of two pinned buffers while the previous slice is on the wire.
static uint64_t stage_slice_bytes() {
    static const uint64_t v = [] { const char* e = getenv("YAMS_B200_STAGE_MIB"); long x = e ? atol(e) : 64; return (uint64_t)(x < 1 ? 1 : x) << 20; }();
    return v;
}
static unsigned stage_threads() {
    static const unsigned v = [] {
        const char* e = getenv("YAMS_B200_STAGE_THREADS");
        long x = e ? atol(e) : (long)std::min(8u, std::max(1u, std::thread::hardware_concurrency()));
        return (unsigned)(x < 1 ? 1 : (x > 64 ? 64 : x));
    }();
    return v;
}
yams_status_t staged_upload(HostBuf pin[2], cudaEvent_t pin_done[2], uint8_t* d_dst, uint64_t total,
                            const std::vector<LayoutPiece>& pieces, cudaStream_t st) {
    if (total == 0) return YAMS_OK;
    yams_status_t rc;
    const uint64_t S = std::min<uint64_t>(stage_slice_bytes(), (total + 255) & ~255ull);
    for (int b = 0; b < 2; ++b)
        if ((rc = pin[b].reserve((size_t)S)) != YAMS_OK) return rc;
    const unsigned T = total < (4u << 20) ? 1u : stage_threads();
    int b = 0;
    for (uint64_t lo = 0; lo < total; lo += S, b ^= 1) {
        const uint64_t hi = std::min<uint64_t>(total, lo + S);
        YB_CUDA(cudaEventSynchronize(pin_done[b]));   // the copy that last used this pinned buffer has finished
        uint8_t* img = pin[b].as<uint8_t>();
        if (T == 1) {
            layout_image(pieces, img, lo, hi);
        } else {
            std::vector<std::thread> th;
            const uint64_t part = (((hi - lo) + T - 1) / T + 4095) & ~4095ull;
            for (unsigned t = 0; t < T; ++t) {
                uint64_t a = lo + (uint64_t)t * part, e = std::min<uint64_t>(hi, a + part);
                if (a < e) th.emplace_back([&pieces, img, lo, a, e] { layout_image(pieces, img + (a - lo), a, e); });
            }
            for (auto& x : th) x.join();
        }
        YB_CUDA(cudaMemcpyAsync(d_dst + lo, img, (size_t)(hi - lo), cudaMemcpyHostToDevice, st));
        YB_CUDA(cudaEventRecord(pin_done[b], st));
    }
    return YAMS_OK;
}
static bool is_pageable(const void* p) {
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        return true;
    }
    return a.type == cudaMemoryTypeUnregistered;
}

// ---- many files per call ----------------------------------------------------------------------------------------
// One group = consecutive files whose padded total fits the staging budget.  Layout: every file starts at a
// 256-byte-aligned buffer position preceded by >= 64 zero bytes, so ONE candidate scan, ONE selection pass and ONE
// SHA-256 launch serve every file of the group.
constexpr uint64_t kBatchGap = 64;
static uint64_t batch_group_bytes() {
    static const uint64_t v = [] { const char* e = getenv("YAMS_B200_BATCH_MIB"); long x = e ? atol(e) : 1024; return (uint64_t)(x < 1 ? 1 : x) << 20; }();
    return v;
}
static inline uint64_t batch_padded(uint64_t len) { return (len + kBatchGap + 255) & ~255ull; }

static yams_status_t run_batch_group(IngestRes& r, const uint8_t* const* files, const size_t* lens, size_t f0, size_t f1,
                                     std::vector<yams_chunk_desc>& out, uint64_t* out_first, float* ms_acc) {
    cudaStream_t st = r.st;
    yams_status_t rc;
    const uint32_t nf = (uint32_t)(f1 - f0);
    std::vector<uint64_t> lay(2 * (size_t)nf);   // starts | ends
    std::vector<LayoutPiece> pieces(nf);
    uint64_t pos = 256;
    for (uint32_t f = 0; f < nf; ++f) {
        lay[f] = pos;
        lay[nf + f] = pos + lens[f0 + f];
        pieces[f] = {pos, lens[f0 + f], files[f0 + f]};
        pos += batch_padded(lens[f0 + f]);
    }
    const uint64_t L = pos;
    if ((rc = r.stage[0].reserve((size_t)L + 256)) != YAMS_OK) return rc;
    uint8_t* d_buf = r.stage[0].as<uint8_t>();
    if ((rc = r.fileinfo.reserve((size_t)nf * 16)) != YAMS_OK) return rc;
    if ((rc = r.first.reserve(((size_t)nf + 1) * 8)) != YAMS_OK) return rc;
    YB_CUDA(cudaEventRecord(r.call[0], st));
    // the whole buffer is uploaded, file bytes and zero gaps alike
    if ((rc = staged_upload(r.pin, r.pin_done, d_buf, L + 256, pieces, st)) != YAMS_OK) return rc;
    YB_CUDA(cudaMemcpyAsync(r.fileinfo.p, lay.data(), (size_t)nf * 16, cudaMemcpyHostToDevice, st));
    YB_CUDA(cudaEventRecord(r.ev[0], st));
    uint32_t ncand = 0;
    if ((rc = r.scan(d_buf, 0, 0, 0, L, &ncand)) != YAMS_OK) return rc;
    YB_CUDA(cudaEventRecord(r.ev[1], st));
    // ---- selection over the merged node table ----
    YB_ARG((uint64_t)ncand + nf < 0xFFFFFFF0ull, "too many nodes in one batch group");
    const BatchArgs B{BatchLayout{r.cand.as<uint64_t>(), ncand, r.fileinfo.as<uint64_t>(), r.fileinfo.as<uint64_t>() + nf, nf, true}, r.P};
    uint64_t nnew = 0;
    if ((rc = r.select_cuts(B, &nnew)) != YAMS_OK) return rc;
    YB_ARG(nnew < 0xFFFFFFFFull, "too many chunks in one batch group");
    if ((rc = r.descs.reserve((size_t)(nnew + 1) * sizeof(yams_chunk_desc))) != YAMS_OK) return rc;
    if ((rc = r.emit_cuts(B, r.descs.as<yams_chunk_desc>())) != YAMS_OK) return rc;
    batch_first_kernel<<<(nf + 1 + 255) / 256, 256, 0, st>>>(B, r.emit_offsets.as<uint32_t>(), r.scalars.as<uint64_t>(),
                                                             r.first.as<uint64_t>());
    YB_CUDA(cudaEventRecord(r.ev[2], st));
    if ((rc = r.hash(d_buf, 0, 0, nnew, L)) != YAMS_OK) return rc;
    YB_CUDA(cudaEventRecord(r.ev[3], st));
    if (nnew) batch_rebase_kernel<<<(unsigned)((nnew + 255) / 256), 256, 0, st>>>(B, r.descs.as<yams_chunk_desc>(), nnew);
    YB_CUDA(cudaGetLastError());
    const size_t base = out.size();
    out.resize(base + (size_t)nnew);
    std::vector<uint64_t> first((size_t)nf + 1);
    if (nnew) YB_CUDA(cudaMemcpyAsync(out.data() + base, r.descs.p, (size_t)nnew * sizeof(yams_chunk_desc), cudaMemcpyDeviceToHost, st));
    YB_CUDA(cudaMemcpyAsync(first.data(), r.first.p, ((size_t)nf + 1) * 8, cudaMemcpyDeviceToHost, st));
    YB_CUDA(cudaEventRecord(r.call[1], st));
    YB_CUDA(cudaStreamSynchronize(st));
    if (out_first)
        for (uint32_t f = 0; f <= nf; ++f) out_first[f0 + f] = base + first[f];
    float a = 0, b = 0, c = 0, d = 0;
    cudaEventElapsedTime(&a, r.ev[0], r.ev[1]);
    cudaEventElapsedTime(&b, r.ev[1], r.ev[2]);
    cudaEventElapsedTime(&c, r.ev[2], r.ev[3]);
    cudaEventElapsedTime(&d, r.call[0], r.call[1]);
    ms_acc[0] += a; ms_acc[1] += b; ms_acc[2] += c; ms_acc[3] += d;
    return YAMS_OK;
}

// SHA-256 of the spans [offsets[i], offsets[i] + sizes[i]) of one buffer; a host buffer is first copied into stage[0].
static yams_status_t hash_spans(const uint8_t* base, bool on_host, size_t base_len, const uint64_t* offsets,
                                const uint64_t* sizes, size_t n, uint8_t* digests) {
    IngestLease ws(nullptr);
    if (ws.rc != YAMS_OK) return ws.rc;
    IngestRes& r = *ws.r;
    if (on_host) {
        yams_status_t rc = r.stage[0].reserve(base_len + 64);
        if (rc != YAMS_OK) return rc;
        if (base_len) YB_CUDA(cudaMemcpyAsync(r.stage[0].p, base, base_len, cudaMemcpyHostToDevice, r.st));
        base = r.stage[0].as<uint8_t>();
    }
    YB_ARG(n < 0xFFFFFFFFull, "too many spans");
    std::vector<yams_chunk_desc> h(n);
    uint64_t total = 0;
    for (size_t i = 0; i < n; ++i) {
        YB_ARG(offsets[i] <= base_len && sizes[i] <= base_len - offsets[i], "span outside the base buffer");
        h[i].offset = offsets[i];
        h[i].size = sizes[i];
        total += sizes[i];
    }
    return r.hash_table(base, h, total, digests);
}

}  // namespace yb

using namespace yb;

// Streaming session: host bytes are staged [carry | slice] into one of two device buffers; the H2D copy
// of slice i+1 overlaps the kernels of slice i (when the host memory is pinned).
struct yams_b200_ingest {
    IngestLease ws;               // held until the session is closed
    bool hash;
    uint64_t head = 0;            // bytes reserved in front of a slice for the carry
    uint64_t stream_pos = 0;      // bytes fed so far
    uint64_t keep_from = 0;       // lowest stream position still resident on the device
    const uint8_t* res_ptr = nullptr;  // device address of stream position keep_from
    int cur = -1;                 // stage buffer holding the resident bytes (-1: none yet)
    bool finished = false;
    float ms_sha = 0;
    uint64_t sha_pos = 0;         // stream position up to which chunks have been hashed (mean chunk size of a slice)
    yams_b200_ingest(const yams_cdc_config* cfg, bool hash_chunks) : ws(cfg), hash(hash_chunks) {}
};

static yams_status_t session_open(const yams_cdc_config* cfg, bool hash, std::unique_ptr<yams_b200_ingest>* out) {
    std::unique_ptr<yams_b200_ingest> s(new (std::nothrow) yams_b200_ingest(cfg, hash));
    if (!s) return YAMS_ERR_INTERNAL;
    if (s->ws.rc != YAMS_OK) return s->ws.rc;
    // the open chunk is always shorter than `force`, and a position needs <= kHistory bytes behind it
    uint64_t need = std::max<uint64_t>(s->ws.r->P.force, (uint64_t)kHistory) + 16;
    s->head = (need + 255) & ~255ull;
    *out = std::move(s);
    return YAMS_OK;
}

static yams_status_t session_sha(yams_b200_ingest* s, const uint8_t* data, uint64_t base_pos, uint64_t first) {
    IngestRes& r = *s->ws.r;
    if (!s->hash || r.ndescs <= first) return YAMS_OK;
    YB_ARG(r.ndescs - first < 0xFFFFFFFFull, "too many chunks in one slice");
    YB_CUDA(cudaEventRecord(r.ev[0], r.st));
    // mean chunk size of the slice: the new chunks end at the open chunk's start
    const uint64_t slice_bytes = r.chunk_start > s->sha_pos ? r.chunk_start - s->sha_pos : 0;
    s->sha_pos = r.chunk_start;
    yams_status_t rc = r.hash(data, base_pos, first, r.ndescs - first, slice_bytes);
    if (rc != YAMS_OK) return rc;
    YB_CUDA(cudaEventRecord(r.ev[1], r.st));
    YB_CUDA(cudaEventSynchronize(r.ev[1]));
    float ms = 0;
    cudaEventElapsedTime(&ms, r.ev[0], r.ev[1]);
    s->ms_sha += ms;
    return YAMS_OK;
}

// Feed `len` host bytes; when `final`, also close the stream.  Newly completed chunks are appended to
// the workspace's descs (digests included when hashing is on).
static yams_status_t session_feed(yams_b200_ingest* s, const uint8_t* data, size_t len, bool final) {
    IngestRes& r = *s->ws.r;
    yams_status_t rc;
    YB_ARG(!s->finished, "ingest session already finished");
    const size_t nslices = (size_t)((len + kFeedSlice - 1) / kFeedSlice);
    if (nslices == 0) {
        if (final) {
            uint64_t first = r.ndescs;
            rc = r.process(s->res_ptr, s->keep_from, s->keep_from, s->stream_pos, s->stream_pos, true);
            if (rc != YAMS_OK) return rc;
            if ((rc = session_sha(s, s->res_ptr, s->keep_from, first)) != YAMS_OK) return rc;
            s->finished = true;
        }
        return YAMS_OK;
    }
    auto slice_len = [&](size_t i) { return (size_t)std::min<uint64_t>(kFeedSlice, (uint64_t)len - i * kFeedSlice); };
    const bool pageable = len >= (4u << 20) && is_pageable(data);
    auto issue_copy = [&](size_t i, int b) -> yams_status_t {
        size_t sl = slice_len(i);
        yams_status_t rr = r.stage[b].reserve((size_t)s->head + sl + 64);
        if (rr != YAMS_OK) return rr;
        YB_CUDA(cudaStreamWaitEvent(r.copy_st, r.freed[b], 0));
        const uint8_t* src = data + i * kFeedSlice;
        if (pageable && sl >= (4u << 20)) {
            // ordinary host memory: pinned double-buffered upload filled by host threads (see staged_upload)
            yams_status_t ur = staged_upload(r.pin, r.pin_done, r.stage[b].as<uint8_t>() + s->head, sl, {{0, (uint64_t)sl, src}}, r.copy_st);
            if (ur != YAMS_OK) return ur;
        } else {
            YB_CUDA(cudaMemcpyAsync(r.stage[b].as<uint8_t>() + s->head, src, sl, cudaMemcpyHostToDevice, r.copy_st));
        }
        YB_CUDA(cudaEventRecord(r.copied[b], r.copy_st));
        return YAMS_OK;
    };
    int b = s->cur < 0 ? 0 : (s->cur ^ 1);
    if ((rc = issue_copy(0, b)) != YAMS_OK) return rc;
    for (size_t i = 0; i < nslices; ++i) {
        const size_t sl = slice_len(i);
        const uint64_t carry = s->stream_pos - s->keep_from;
        uint8_t* dst0 = r.stage[b].as<uint8_t>() + s->head;  // device address of stream position stream_pos
        if (carry) {
            YB_CUDA(cudaMemcpyAsync(dst0 - carry, s->res_ptr, (size_t)carry, cudaMemcpyDeviceToDevice, r.st));
        }
        if (s->cur >= 0) YB_CUDA(cudaEventRecord(r.freed[s->cur], r.st));
        if (i + 1 < nslices) {
            if ((rc = issue_copy(i + 1, b ^ 1)) != YAMS_OK) return rc;
        }
        YB_CUDA(cudaStreamWaitEvent(r.st, r.copied[b], 0));
        const uint64_t new_pos = s->stream_pos + sl;
        const uint64_t first = r.ndescs;
        const uint8_t* view = dst0 - carry;  // stream position keep_from
        const bool last = final && (i + 1 == nslices);
        rc = r.process(view, s->keep_from, s->keep_from, s->stream_pos, new_pos, last);
        if (rc != YAMS_OK) return rc;
        if ((rc = session_sha(s, view, s->keep_from, first)) != YAMS_OK) return rc;
        s->stream_pos = new_pos;
        uint64_t nk = std::min<uint64_t>(r.chunk_start, new_pos > (uint64_t)kHistory ? new_pos - kHistory : 0);
        if (nk < s->keep_from) nk = s->keep_from;
        s->res_ptr = view + (nk - s->keep_from);
        s->keep_from = nk;
        s->cur = b;
        b ^= 1;
    }
    if (final) s->finished = true;
    return YAMS_OK;
}

static yams_status_t session_take(yams_b200_ingest* s, yams_chunk_desc** out, size_t* out_n) {
    IngestRes& r = *s->ws.r;
    yams_status_t rc = copy_out(r, 0, r.ndescs, out, out_n);
    if (rc == YAMS_OK) r.ndescs = 0;  // descriptors handed over; reuse the device table
    return rc;
}

static yams_status_t run_host(const uint8_t* data, size_t len, const yams_cdc_config* cfg, bool hash,
                              yams_chunk_desc** out, size_t* out_n) {
    std::unique_ptr<yams_b200_ingest> s;
    yams_status_t rc = session_open(cfg, hash, &s);
    if (rc != YAMS_OK) return rc;
    IngestRes& r = *s->ws.r;
    if ((rc = r.presize_descs(len)) != YAMS_OK) return rc;
    YB_CUDA(cudaEventRecord(r.call[0], r.st));
    if ((rc = session_feed(s.get(), data, len, true)) != YAMS_OK) return rc;
    if ((rc = session_take(s.get(), out, out_n)) != YAMS_OK) return rc;
    YB_CUDA(cudaEventRecord(r.call[1], r.st));
    YB_CUDA(cudaEventSynchronize(r.call[1]));
    float t = 0;
    cudaEventElapsedTime(&t, r.call[0], r.call[1]);
    report_timings({r.ms_scan, r.ms_select, s->ms_sha, t}, &r);
    return YAMS_OK;
}

extern "C" {

void yams_b200_cdc_default_config(yams_cdc_config* cfg) {
    // /root/reference/include/yams/chunking/chunker.h:44-51, include/yams/core/types.h:280-285;
    // `yams add` uses StreamingChunker: src/api/content_store_builder.cpp:152-165
    if (!cfg) return;
    cfg->window_size = 48;
    cfg->min_chunk = 16 * 1024;
    cfg->max_chunk = 1024 * 1024;
    cfg->polynomial = kDefaultPoly;
    cfg->mask = 0x1FFF;
    cfg->variant = YAMS_CDC_STREAMING;
    cfg->reserved = 0;
}

yams_status_t yams_b200_chunk_and_hash(void* self, const uint8_t* data, size_t len, const yams_cdc_config* cfg,
                                       yams_chunk_desc** out, size_t* out_n) {
    YB_TRY
    (void)self;
    YB_ARG(out && out_n, "out / out_n is null");
    *out = nullptr;
    *out_n = 0;
    YB_ARG(data || len == 0, "data is null");
    YB_ARG(cfg, "cfg is null");
    return run_host(data, len, cfg, true, out, out_n);
    YB_CATCH
}

yams_status_t yams_b200_chunk_boundaries(void* self, const uint8_t* data, size_t len, const yams_cdc_config* cfg,
                                         yams_chunk_desc** out, size_t* out_n) {
    YB_TRY
    (void)self;
    YB_ARG(out && out_n, "out / out_n is null");
    *out = nullptr;
    *out_n = 0;
    YB_ARG(data || len == 0, "data is null");
    YB_ARG(cfg, "cfg is null");
    yams_status_t rc = run_host(data, len, cfg, false, out, out_n);
    if (rc == YAMS_OK)
        for (size_t i = 0; i < *out_n; ++i) memset((*out)[i].digest, 0, 32);
    return rc;
    YB_CATCH
}

yams_status_t yams_b200_chunk_and_hash_device(void* self, const uint8_t* d_data, size_t len,
                                              const yams_cdc_config* cfg, yams_chunk_desc** out, size_t* out_n) {
    YB_TRY
    (void)self;
    YB_ARG(out && out_n, "out / out_n is null");
    *out = nullptr;
    *out_n = 0;
    YB_ARG(d_data || len == 0, "d_data is null");
    YB_ARG(cfg, "cfg is null");
    return run_device(d_data, len, cfg, out, out_n);
    YB_CATCH
}

yams_status_t yams_b200_chunk_and_hash_batch(void* self, const uint8_t* const* files, const size_t* lens, size_t n_files,
                                             const yams_cdc_config* cfg, yams_chunk_desc** out, size_t* out_n, uint64_t* out_first) {
    YB_TRY
    (void)self;
    YB_ARG(out && out_n, "out / out_n is null");
    *out = nullptr;
    *out_n = 0;
    YB_ARG(cfg, "cfg is null");
    if (out_first) out_first[0] = 0;
    if (n_files == 0) return YAMS_OK;
    YB_ARG(files && lens && out_first, "null argument");
    for (size_t f = 0; f < n_files; ++f) YB_ARG(files[f] || lens[f] == 0, "a file pointer is null");
    IngestLease ws(cfg);
    if (ws.rc != YAMS_OK) return ws.rc;
    yams_status_t rc;
    std::vector<yams_chunk_desc> all;
    float ms[4] = {0, 0, 0, 0};
    const uint64_t budget = batch_group_bytes();
    size_t f = 0;
    while (f < n_files) {
        if (batch_padded(lens[f]) + 256 > budget) {
            // a file larger than a whole group goes through the streaming path on its own
            yams_chunk_desc* d = nullptr;
            size_t n = 0;
            if ((rc = run_host(files[f], lens[f], cfg, true, &d, &n)) != YAMS_OK) return rc;
            out_first[f] = all.size();
            all.insert(all.end(), d, d + n);
            out_first[f + 1] = all.size();
            free(d);
            for (int i = 0; i < 4; ++i) ms[i] += g_last_ms[i];
            ++f;
            continue;
        }
        size_t g = f;
        uint64_t tot = 256;
        while (g < n_files && tot + batch_padded(lens[g]) <= budget) tot += batch_padded(lens[g++]);
        if ((rc = run_batch_group(*ws.r, files, lens, f, g, all, out_first, ms)) != YAMS_OK) return rc;
        f = g;
    }
    report_timings(ms, nullptr);
    if (!all.empty()) {
        yams_chunk_desc* h = static_cast<yams_chunk_desc*>(malloc(all.size() * sizeof(yams_chunk_desc)));
        if (!h) {
            set_last_error("out of host memory for %llu chunk descriptors", (unsigned long long)all.size());
            return YAMS_ERR_INTERNAL;
        }
        memcpy(h, all.data(), all.size() * sizeof(yams_chunk_desc));
        *out = h;
        *out_n = all.size();
    }
    return YAMS_OK;
    YB_CATCH
}

void yams_b200_free_chunks(void* self, yams_chunk_desc* chunks, size_t n) {
    (void)self;
    (void)n;
    free(chunks);
}

yams_status_t yams_b200_ingest_open(void* self, const yams_cdc_config* cfg, yams_b200_ingest** out) {
    YB_TRY
    (void)self;
    YB_ARG(out, "out is null");
    *out = nullptr;
    YB_ARG(cfg, "cfg is null");
    std::unique_ptr<yams_b200_ingest> s;
    yams_status_t rc = session_open(cfg, true, &s);
    if (rc == YAMS_OK) *out = s.release();
    return rc;
    YB_CATCH
}

yams_status_t yams_b200_ingest_feed(yams_b200_ingest* s, const uint8_t* data, size_t len, yams_chunk_desc** out,
                                    size_t* out_n) {
    YB_TRY
    YB_ARG(s && out && out_n, "null argument");
    cudaSetDevice(s->ws.r->dev->device);   // a session may be fed from another thread than the one that opened it
    *out = nullptr;
    *out_n = 0;
    YB_ARG(data || len == 0, "data is null");
    yams_status_t rc = session_feed(s, data, len, false);
    if (rc != YAMS_OK) return rc;
    return session_take(s, out, out_n);
    YB_CATCH
}

yams_status_t yams_b200_ingest_finish(yams_b200_ingest* s, yams_chunk_desc** out, size_t* out_n) {
    YB_TRY
    YB_ARG(s && out && out_n, "null argument");
    cudaSetDevice(s->ws.r->dev->device);   // a session may be fed from another thread than the one that opened it
    *out = nullptr;
    *out_n = 0;
    yams_status_t rc = session_feed(s, nullptr, 0, true);
    if (rc != YAMS_OK) return rc;
    return session_take(s, out, out_n);
    YB_CATCH
}

void yams_b200_ingest_close(yams_b200_ingest* s) { delete s; }

yams_status_t yams_b200_sha256_batch_device(void* self, const uint8_t* d_base, size_t base_len,
                                            const uint64_t* offsets, const uint64_t* sizes, size_t n,
                                            uint8_t* digests) {
    YB_TRY
    (void)self;
    if (n == 0) return YAMS_OK;
    YB_ARG(offsets && sizes && digests, "null argument");
    YB_ARG(d_base || base_len == 0, "d_base is null");
    return hash_spans(d_base, false, base_len, offsets, sizes, n, digests);
    YB_CATCH
}

yams_status_t yams_b200_sha256_batch(void* self, const uint8_t* base, size_t base_len, const uint64_t* offsets,
                                     const uint64_t* sizes, size_t n, uint8_t* digests) {
    YB_TRY
    (void)self;
    if (n == 0) return YAMS_OK;
    YB_ARG(offsets && sizes && digests, "null argument");
    YB_ARG(base || base_len == 0, "base is null");
    return hash_spans(base, true, base_len, offsets, sizes, n, digests);
    YB_CATCH
}

// Many separate messages (IContentHasher::hash per span, ChunkValidator::validateChunks): packed 16-byte aligned into
// the pooled staging buffer by the pinned upload path, hashed by one launch per <= 1 GiB group.
yams_status_t yams_b200_sha256_many(void* self, const uint8_t* const* msgs, const size_t* lens, size_t n, uint8_t* digests) {
    YB_TRY
    (void)self;
    if (n == 0) return YAMS_OK;
    YB_ARG(msgs && lens && digests, "null argument");
    for (size_t i = 0; i < n; ++i) YB_ARG(msgs[i] || lens[i] == 0, "a message pointer is null");
    yams_cdc_config cfg;
    yams_b200_cdc_default_config(&cfg);
    IngestLease ws(&cfg);
    if (ws.rc != YAMS_OK) return ws.rc;
    IngestRes& r = *ws.r;
    yams_status_t rc;
    const uint64_t budget = batch_group_bytes();
    for (size_t i0 = 0, i1; i0 < n; i0 = i1) {
        // group [i0, i1): packed size within the budget (a single larger message forms its own group)
        i1 = i0;
        uint64_t tot = 0;
        std::vector<yams_chunk_desc> h;
        std::vector<LayoutPiece> pieces;
        while (i1 < n && (i1 == i0 || tot + lens[i1] + 16 <= budget) && h.size() < 0xFFFFFFF0ull) {
            yams_chunk_desc d{};
            d.offset = tot;
            d.size = lens[i1];
            h.push_back(d);
            pieces.push_back({tot, lens[i1], msgs[i1]});
            tot = (tot + lens[i1] + 15) & ~15ull;
            ++i1;
        }
        if ((rc = r.stage[0].reserve((size_t)tot + 256)) != YAMS_OK) return rc;
        if ((rc = staged_upload(r.pin, r.pin_done, r.stage[0].as<uint8_t>(), tot, pieces, r.st)) != YAMS_OK) return rc;
        if ((rc = r.hash_table(r.stage[0].as<uint8_t>(), h, tot, digests + 32 * i0)) != YAMS_OK) return rc;
    }
    return YAMS_OK;
    YB_CATCH
}

yams_status_t yams_b200_dedup_stats(void* self, const yams_chunk_desc* chunks, size_t n, yams_dedup_stats* out) {
    YB_TRY
    (void)self;
    YB_ARG(out, "out is null");
    memset(out, 0, sizeof(*out));
    if (n == 0) return YAMS_OK;
    YB_ARG(chunks, "chunks is null");
    YB_ARG(n < (1ull << 31), "too many chunks");
    DeviceCtx* dev = nullptr;
    yams_status_t rc = ensure_device(&dev);
    if (rc != YAMS_OK) return rc;
    cudaStream_t st;
    YB_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    uint64_t slots = 1;
    while (slots < 2 * (uint64_t)n) slots <<= 1;   // load factor <= 0.5
    DevBuf d_descs, d_table, d_out;
    rc = d_descs.reserve(n * sizeof(yams_chunk_desc));
    if (rc == YAMS_OK) rc = d_table.reserve(slots * 4);
    if (rc == YAMS_OK) rc = d_out.reserve(sizeof(yams_dedup_stats));
    if (rc == YAMS_OK) {
        cudaMemcpyAsync(d_descs.p, chunks, n * sizeof(yams_chunk_desc), cudaMemcpyHostToDevice, st);
        cudaMemsetAsync(d_table.p, 0xFF, slots * 4, st);
        cudaMemsetAsync(d_out.p, 0, sizeof(yams_dedup_stats), st);
        rc = launch_dedup_stats(d_descs.as<yams_chunk_desc>(), (uint32_t)n, d_table.as<uint32_t>(), slots,
                                reinterpret_cast<unsigned long long*>(d_out.p), st);
        if (rc == YAMS_OK) {
            cudaError_t e = cudaMemcpyAsync(out, d_out.p, sizeof(yams_dedup_stats), cudaMemcpyDeviceToHost, st);
            if (e == cudaSuccess) e = cudaStreamSynchronize(st);
            if (e != cudaSuccess) {
                set_last_error("dedup_stats failed: %s", cudaGetErrorString(e));
                rc = YAMS_ERR_INTERNAL;
            }
        }
    }
    cudaStreamDestroy(st);
    return rc;
    YB_CATCH
}

yams_status_t yams_b200_ingest_last_timings(void* self, float out_ms[8]) {
    (void)self;
    YB_ARG(out_ms, "out_ms is null");
    for (int i = 0; i < 8; ++i) out_ms[i] = g_last_ms[i];
    return YAMS_OK;
}

// bench / test utility: SURVEY.md §8d byte stream generated straight into HBM
yams_status_t yams_b200_synth_bytes_device(uint64_t seed, uint64_t start, uint64_t n, uint8_t* d_out) {
    DeviceCtx* dev = nullptr;
    yams_status_t rc = ensure_device(&dev);
    if (rc != YAMS_OK) return rc;
    YB_ARG(d_out || n == 0, "d_out is null");
    rc = launch_synth_bytes(seed, start, n, d_out, dev->sm_count, 0);
    if (rc != YAMS_OK) return rc;
    YB_CUDA(cudaStreamSynchronize(0));
    return YAMS_OK;
}

}  // extern "C"
