// api.cu -- plugin envelope (abi.h:17-33 conventions), device context, error plumbing, the pooled operator workspace
// (OpWs) and the health JSON of libyams_b200.so.
#include <stdarg.h>
#include <stdlib.h>

#include <mutex>

#include <vector>

#include "common.cuh"

namespace yb {

static thread_local char g_tls_error[512] = "";
static std::mutex g_mu;
static char g_global_error[512] = "";
static DeviceCtx g_dev;
static int g_requested_device = -1;
static bool g_inited = false;
std::atomic<uint64_t> g_device_buffer_bytes{0}, g_pinned_buffer_bytes{0};

void set_last_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_tls_error, sizeof g_tls_error, fmt, ap);
    va_end(ap);
    note_global_error(g_tls_error);
}
const char* last_error() { return g_tls_error; }
void note_global_error(const char* text) {
    std::lock_guard<std::mutex> lk(g_mu);
    snprintf(g_global_error, sizeof g_global_error, "%s", text);
}
void set_requested_device(int dev) { g_requested_device = dev; }

yams_status_t ensure_device(DeviceCtx** out) {
    std::lock_guard<std::mutex> lk(g_mu);
    if (!g_dev.ok) {
        int n = 0;
        cudaError_t e = cudaGetDeviceCount(&n);
        if (e != cudaSuccess || n == 0) {
            snprintf(g_tls_error, sizeof g_tls_error,
                     "no CUDA device available (%s); libyams_b200 has no CPU fallback",
                     e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
            snprintf(g_global_error, sizeof g_global_error, "%s", g_tls_error);
            return YAMS_ERR_INTERNAL;
        }
        int dev = g_requested_device;
        if (dev < 0) {
            const char* lr = getenv("LOCAL_RANK");
            dev = lr ? atoi(lr) : 0;
        }
        if (dev >= n) dev = dev % n;
        cudaDeviceProp prop;
        if ((e = cudaSetDevice(dev)) != cudaSuccess || (e = cudaGetDeviceProperties(&prop, dev)) != cudaSuccess) {
            snprintf(g_tls_error, sizeof g_tls_error, "cudaSetDevice(%d) failed: %s", dev, cudaGetErrorString(e));
            snprintf(g_global_error, sizeof g_global_error, "%s", g_tls_error);
            return YAMS_ERR_INTERNAL;
        }
        if (prop.major != 9 || prop.minor != 0) {
            snprintf(g_tls_error, sizeof g_tls_error,
                     "device %d is sm_%d%d; libyams_b200 is built for sm_90a (H100) only", dev, prop.major,
                     prop.minor);
            snprintf(g_global_error, sizeof g_global_error, "%s", g_tls_error);
            return YAMS_ERR_INTERNAL;
        }
        g_dev.device = dev;
        g_dev.sm_count = prop.multiProcessorCount;
        g_dev.cc_major = prop.major;
        g_dev.cc_minor = prop.minor;
        g_dev.ok = true;
    } else {
        // other host threads must bind the same device
        cudaSetDevice(g_dev.device);
    }
    *out = &g_dev;
    return YAMS_OK;
}

static std::mutex g_ws_mu;
static std::vector<OpWs*> g_ws_free;

OpWs* opws_acquire() {
    DeviceCtx* dev = nullptr;
    if (ensure_device(&dev) != YAMS_OK) return nullptr;   // also binds the device on this thread
    {
        std::lock_guard<std::mutex> lk(g_ws_mu);
        if (!g_ws_free.empty()) {
            OpWs* w = g_ws_free.back();
            g_ws_free.pop_back();
            return w;
        }
    }
    OpWs* w = new (std::nothrow) OpWs();
    if (!w) return nullptr;
    if (cudaStreamCreateWithFlags(&w->st, cudaStreamNonBlocking) != cudaSuccess) {
        set_last_error("cudaStreamCreate failed");
        delete w;
        return nullptr;
    }
    return w;
}
void opws_release(OpWs* w) {
    std::lock_guard<std::mutex> lk(g_ws_mu);
    if (g_ws_free.size() < 16) {
        g_ws_free.push_back(w);
        return;
    }
    delete w;
}

}  // namespace yb

using namespace yb;

// vtables are filled once; the functions are the exported C symbols themselves
static yams_content_ingest_v1 g_ingest_vt;
static yams_vector_scan_v1 g_scan_vt;

extern "C" {

int yams_plugin_get_abi_version(void) { return YAMS_PLUGIN_ABI_VERSION; }
const char* yams_plugin_get_name(void) { return "yams_b200"; }
const char* yams_plugin_get_version(void) { return "0.1.0"; }
const char* yams_plugin_get_manifest_json(void) {
    return "{\"name\": \"yams_b200\", \"version\": \"0.1.0\", \"abi\": 1, "
           "\"interfaces\": [{\"id\": \"vector_scan_v1\", \"version\": 1}, "
           "{\"id\": \"content_ingest_v1\", \"version\": 1}]}";
}

int yams_plugin_init(const char* config_json, const void* host_context) {
    (void)host_context;
    if (config_json) {
        const char* p = strstr(config_json, "\"device\"");
        if (p && (p = strchr(p, ':'))) set_requested_device(atoi(p + 1));
    }
    g_ingest_vt.abi_version = YAMS_IFACE_CONTENT_INGEST_V1_VERSION;
    g_ingest_vt.self = nullptr;
    g_ingest_vt.chunk_and_hash = yams_b200_chunk_and_hash;
    g_ingest_vt.free_chunks = yams_b200_free_chunks;
    g_ingest_vt.ingest_open = yams_b200_ingest_open;
    g_ingest_vt.ingest_feed = yams_b200_ingest_feed;
    g_ingest_vt.ingest_finish = yams_b200_ingest_finish;
    g_ingest_vt.ingest_close = yams_b200_ingest_close;
    g_ingest_vt.sha256_batch = yams_b200_sha256_batch;
    g_ingest_vt.dedup_stats = yams_b200_dedup_stats;
    g_ingest_vt.chunk_and_hash_batch = yams_b200_chunk_and_hash_batch;
    g_ingest_vt.sha256_many = yams_b200_sha256_many;
    g_ingest_vt.digest_set_create = yams_b200_digest_set_create;
    g_ingest_vt.digest_set_insert = yams_b200_digest_set_insert;
    g_ingest_vt.digest_set_contains = yams_b200_digest_set_contains;
    g_ingest_vt.digest_set_size = yams_b200_digest_set_size;
    g_ingest_vt.digest_set_destroy = yams_b200_digest_set_destroy;
    g_ingest_vt.manifest_build = yams_b200_manifest_build;
    g_scan_vt.abi_version = YAMS_IFACE_VECTOR_SCAN_V1_VERSION;
    g_scan_vt.self = nullptr;
    g_scan_vt.corpus_create = yams_b200_corpus_create;
    g_scan_vt.corpus_append = yams_b200_corpus_append;
    g_scan_vt.corpus_clear = yams_b200_corpus_clear;
    g_scan_vt.corpus_size = yams_b200_corpus_size;
    g_scan_vt.corpus_destroy = yams_b200_corpus_destroy;
    g_scan_vt.search = yams_b200_search;
    g_scan_vt.vec0_exact = yams_b200_vec0_exact;
    g_scan_vt.corpus_remove = yams_b200_corpus_remove;
    g_scan_vt.search_all_matching = yams_b200_search_all_matching;
    g_scan_vt.batch_distance = yams_b200_batch_distance;
    g_scan_vt.compute_cosine_similarity = yams_b200_compute_cosine_similarity;
    g_scan_vt.compute_cosine_similarity_many = yams_b200_compute_cosine_similarity_many;
    g_scan_vt.search_exhaustive = yams_b200_search_exhaustive;
    g_scan_vt.pq_build = yams_b200_pq_build;
    g_scan_vt.pq_search = yams_b200_pq_search;
    g_scan_vt.pq_destroy = yams_b200_pq_destroy;
    g_scan_vt.pq_search_candidates = yams_b200_pq_search_candidates;
    g_scan_vt.search_documents = yams_b200_search_documents;
    g_scan_vt.semantic_neighbors = yams_b200_semantic_neighbors;
    DeviceCtx* dev = nullptr;
    if (ensure_device(&dev) != YAMS_OK) return YAMS_PLUGIN_ERR_INIT_FAILED;  // no CPU fallback
    g_inited = true;
    return YAMS_PLUGIN_OK;
}

void yams_plugin_shutdown(void) { g_inited = false; }

int yams_plugin_get_interface(const char* iface_id, uint32_t version, void** out_iface) {
    if (!iface_id || !out_iface) return YAMS_PLUGIN_ERR_INVALID;
    *out_iface = nullptr;
    if (!g_inited) return YAMS_PLUGIN_ERR_INIT_FAILED;
    if (strcmp(iface_id, YAMS_IFACE_VECTOR_SCAN_V1) == 0) {
        if (version != YAMS_IFACE_VECTOR_SCAN_V1_VERSION) return YAMS_PLUGIN_ERR_NOT_FOUND;
        *out_iface = &g_scan_vt;
        return YAMS_PLUGIN_OK;
    }
    if (strcmp(iface_id, YAMS_IFACE_CONTENT_INGEST_V1) == 0) {
        if (version != YAMS_IFACE_CONTENT_INGEST_V1_VERSION) return YAMS_PLUGIN_ERR_NOT_FOUND;
        *out_iface = &g_ingest_vt;
        return YAMS_PLUGIN_OK;
    }
    return YAMS_PLUGIN_ERR_NOT_FOUND;
}

int yams_plugin_get_health_json(char** out_json) {
    if (!out_json) return YAMS_PLUGIN_ERR_INVALID;
    char buf[1024];
    std::lock_guard<std::mutex> lk(g_mu);
    // escape quotes / backslashes of the error text
    char esc[600];
    size_t j = 0;
    for (size_t i = 0; g_global_error[i] && j + 2 < sizeof esc; ++i) {
        char c = g_global_error[i];
        if (c == '"' || c == '\\') esc[j++] = '\\';
        esc[j++] = (c == '\n') ? ' ' : c;
    }
    esc[j] = 0;
    snprintf(buf, sizeof buf,
             "{\"status\": \"%s\", \"device\": %d, \"sm_count\": %d, \"compute_capability\": \"%d.%d\", "
             "\"device_buffer_bytes\": %llu, \"pinned_buffer_bytes\": %llu, \"last_error\": \"%s\"}",
             g_dev.ok ? "ok" : (g_inited ? "degraded" : "uninitialized"), g_dev.device, g_dev.sm_count,
             g_dev.cc_major, g_dev.cc_minor, (unsigned long long)g_device_buffer_bytes.load(),
             (unsigned long long)g_pinned_buffer_bytes.load(), esc);
    *out_json = strdup(buf);
    return *out_json ? YAMS_PLUGIN_OK : YAMS_PLUGIN_ERR_INVALID;
}

int yams_b200_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}
const char* yams_b200_last_error(void) { return last_error(); }

}  // extern "C"
