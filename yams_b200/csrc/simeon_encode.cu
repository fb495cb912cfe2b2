// simeon_encode.cu -- the Simeon text encoder on the device: the two profiles YAMS runs (SURVEY.md §8f N4).
//
// Reference (paths under /root/reference/third_party/simeon):
//   Encoder::Impl::encode_one                       src/simeon.cpp:190-262
//   emit_char_ngrams (CharOnly, Text scope)         src/tokenizer.cpp:25-38
//   splitmix64_hash                                 src/hasher.cpp:33-47, include/simeon/hasher.hpp:12-16
//   SketchSink (integer count sketch, +-2 per gram) src/simeon.cpp:355-373, sketch_bucket :46-49
//   Projection (AchlioptasSparse)                   src/projection.cpp:22-34 (entry), :326-343 (apply: int64 pos - neg, one float scale)
//   simd::l2_normalize, AVX2 tier                   src/arch/avx2.cpp:31-60
//   emit_word_tokens (CharAndWord)                  src/tokenizer.cpp:40-52 (one +-1 feature per [A-Za-z0-9_]+ run)
//   Projection (Fwht)                               src/projection.cpp:149-186 (signs, row sample), :359-374 (apply), fwht_inplace :50-70
//   the profiles YAMS runs: `simeon-v1-384` = CharOnly + AchlioptasSparse (src/simeon.cpp:75-93); the "configurable" default of an
//   unconfigured [embeddings.simeon] = CharAndWord + Fwht, sketch 4096, output = embedding_dim
//   (/root/reference/src/embedding_simeon/simeon_embedding_backend.cpp:18-47,118-135)
//
// Everything up to the projection is integer arithmetic: every byte n-gram of length ngram_min..ngram_max is hashed
// (splitmix64 over little-endian 8-byte words + a length-tagged tail), the low hash bits pick one of sketch_dim buckets, the top
// bit the sign, and +-2 is added (integer atomics in shared memory: order-free, exact).  The Achlioptas matrix entry of (row, col)
// is a hash of the pair: -1 with probability 1/6, +1 with 1/6; the reference sums the sketch values under each sign in int64 and
// multiplies ONCE by sqrt(3)/sqrt(output_dim) in float.  Only the L2 normalisation is a float reduction; it follows the lane
// structure of the AVX2 kernel.  The output is therefore bit-identical to the reference encoder
// (tests/test_gpu_simeon.py pins it against simeon's own sources compiled in place; tests/test_gpu_simeon_restated.py against a
// numpy restatement of the encoder at any configuration).
// Fwht: the sketch, zero-padded to a power of two and multiplied by a +-1 diagonal, goes through the in-place Walsh-Hadamard
// butterflies in shared memory (same stage order and the same x + y / x - y per butterfly as fwht_inplace, so every float is the
// reference's), output_dim sampled coordinates are scaled by 1/sqrt(output_dim).
//
// One CTA per text.  The sign matrix is tabulated once per encoder, 2 bits per entry, column-major (for one sketch column the
// 384 row signs are 96 contiguous bytes): the projection walks the NON-ZERO sketch columns only.
#include <algorithm>
#include <memory>
#include <mutex>
#include <new>
#include <vector>

#include "common.cuh"
#include "text_hash.cuh"

namespace yb {

constexpr int ENC_THREADS = 256;

// achlioptas_entry (projection.cpp:22-34) as a 2-bit code: 0 zero, 1 plus, 2 minus
__global__ void achlioptas_table_kernel(uint32_t sketch_dim, uint32_t output_dim, uint64_t seed, uint32_t words_per_col, uint32_t* __restrict__ table) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (uint64_t)sketch_dim * words_per_col) return;
    const uint32_t col = (uint32_t)(t / words_per_col), w = (uint32_t)(t % words_per_col);
    uint32_t packed = 0;
    for (uint32_t b = 0; b < 16; ++b) {
        const uint32_t row = w * 16 + b;
        if (row >= output_dim) break;
        const uint64_t key = ((uint64_t)row << 32) ^ (uint64_t)col;
        const uint64_t h = sm64_mix(key ^ seed);
        uint32_t code = 0;
        if (h < 0x2AAAAAAAAAAAAAABULL) code = 2;
        else if (h >= 0xD555555555555555ULL) code = 1;
        packed |= code << (2 * b);
    }
    table[t] = packed;
}

struct EncArgs {
    const uint8_t* text;        // all texts back to back
    const uint64_t* offsets;    // n + 1
    uint32_t n;
    uint32_t kmin, kmax, sketch_dim, output_dim, words_per_col;
    uint64_t h0;                // gram_hash_h0(hash_seed)
    const uint32_t* table;
    float scale;                // sqrt(3.0f) * (1.0f / sqrt((float)output_dim)), evaluated on the host in float like projection.cpp:128-129
    int l2_normalize;
    float* out;                 // n x output_dim
    uint32_t flags;             // YAMS_SIMEON_WORD_TOKENS | YAMS_SIMEON_PROJECTION_FWHT
    uint32_t pad_n;             // Fwht: next_pow2(sketch_dim)
    const float* signs;         // Fwht: pad_n entries of +-1
    const uint32_t* sample;     // Fwht: output_dim distinct coordinates of the transformed vector
    float fwht_scale;           // Fwht: 1.0f / sqrt((float)output_dim)
};

__global__ void __launch_bounds__(ENC_THREADS) simeon_encode_kernel(EncArgs a) {
    extern __shared__ unsigned char sm[];
    int32_t* sketch = reinterpret_cast<int32_t*>(sm);                      // sketch_dim
    uint32_t* nz = reinterpret_cast<uint32_t*>(sketch + a.sketch_dim);     // sketch_dim: compacted non-zero columns (Achlioptas)
    float* wh = reinterpret_cast<float*>(nz);                              // pad_n: Walsh-Hadamard buffer (Fwht) -- same region
    const uint32_t region2 = a.pad_n > a.sketch_dim ? a.pad_n : a.sketch_dim;
    float* outv = reinterpret_cast<float*>(nz + region2);                  // output_dim
    __shared__ uint32_t s_nnz;
    __shared__ float s_inv;
    __shared__ int s_scale;
    for (uint32_t t = blockIdx.x; t < a.n; t += gridDim.x) {
        const uint8_t* p = a.text + a.offsets[t];
        const uint64_t len = a.offsets[t + 1] - a.offsets[t];
        for (uint32_t i = threadIdx.x; i < a.sketch_dim; i += ENC_THREADS) sketch[i] = 0;
        if (threadIdx.x == 0) s_nnz = 0;
        __syncthreads();
        // ---- count sketch of every byte n-gram (tokenizer.cpp:25-38, simeon.cpp:355-373) ----
        for (uint32_t k = a.kmin; k <= a.kmax; ++k) {
            if (len < k) break;
            const uint64_t last = len - k;
            for (uint64_t i = threadIdx.x; i <= last; i += ENC_THREADS) {
                const uint64_t h = gram_hash(p + i, k, a.h0);
                const uint32_t low = (uint32_t)h;
                const uint32_t bucket = (a.sketch_dim & (a.sketch_dim - 1)) == 0 ? (low & (a.sketch_dim - 1)) : (low % a.sketch_dim);
                atomicAdd(&sketch[bucket], (h >> 63) ? -2 : 2);            // char n-grams weigh 1.0 -> magnitude 2
            }
        }
        // ---- word tokens (tokenizer.cpp:40-52): every maximal [A-Za-z0-9_]+ run is one feature of weight 0.5 -> magnitude 1;
        //      the thread that sees a run's first byte hashes the whole run ----
        if (a.flags & YAMS_SIMEON_WORD_TOKENS) {
            for (uint64_t i = threadIdx.x; i < len; i += ENC_THREADS) {
                if (!is_word_char(p[i]) || (i > 0 && is_word_char(p[i - 1]))) continue;
                uint64_t e = i + 1;
                while (e < len && is_word_char(p[e])) ++e;
                const uint64_t h = gram_hash(p + i, (uint32_t)(e - i), a.h0);
                const uint32_t low = (uint32_t)h;
                const uint32_t bucket = (a.sketch_dim & (a.sketch_dim - 1)) == 0 ? (low & (a.sketch_dim - 1)) : (low % a.sketch_dim);
                atomicAdd(&sketch[bucket], (h >> 63) ? -1 : 1);
            }
        }
        __syncthreads();
        if (a.flags & YAMS_SIMEON_PROJECTION_FWHT) {
            // ---- Fwht (projection.cpp:359-374): pad, sign diagonal, in-place butterflies, sample, scale ----
            for (uint32_t i = threadIdx.x; i < a.pad_n; i += ENC_THREADS)
                wh[i] = i < a.sketch_dim ? __fmul_rn((float)sketch[i], __ldg(&a.signs[i])) : 0.0f;
            __syncthreads();
            for (uint32_t h = 1; h < a.pad_n; h <<= 1) {
                for (uint32_t tb = threadIdx.x; tb < a.pad_n / 2; tb += ENC_THREADS) {
                    const uint32_t j = (tb / h) * (h << 1) + (tb % h);
                    const float x = wh[j], y = wh[j + h];
                    wh[j] = __fadd_rn(x, y);
                    wh[j + h] = __fsub_rn(x, y);
                }
                __syncthreads();
            }
            for (uint32_t row = threadIdx.x; row < a.output_dim; row += ENC_THREADS)
                outv[row] = __fmul_rn(wh[__ldg(&a.sample[row])], a.fwht_scale);
        } else {
        // ---- non-zero columns, ascending order is irrelevant for an integer sum ----
        for (uint32_t i = threadIdx.x; i < a.sketch_dim; i += ENC_THREADS)
            if (sketch[i] != 0) nz[atomicAdd(&s_nnz, 1u)] = i;
        __syncthreads();
        const uint32_t nnz = s_nnz;
        // ---- Achlioptas projection: int64 (sum under +) - (sum under -), one float scale (projection.cpp:326-343) ----
        for (uint32_t row = threadIdx.x; row < a.output_dim; row += ENC_THREADS) {
            long long pos = 0, neg = 0;
            const uint32_t w = row >> 4, sh = (row & 15) * 2;
            for (uint32_t j = 0; j < nnz; ++j) {
                const uint32_t col = nz[j];
                const uint32_t code = (__ldg(&a.table[(size_t)col * a.words_per_col + w]) >> sh) & 3u;
                const long long v = sketch[col];
                if (code == 1) pos += v;
                else if (code == 2) neg += v;
            }
            outv[row] = __fmul_rn((float)(pos - neg), a.scale);
        }
        }
        __syncthreads();
        // ---- simd::l2_normalize, AVX2 tier (avx2.cpp:31-60): two 8-lane FMA accumulators over 16-element blocks ----
        if (a.l2_normalize) {
            if (threadIdx.x < 32) {
                const uint32_t lane = threadIdx.x;
                const uint32_t n16 = a.output_dim & ~15u;
                float acc = 0.f;                                            // lanes 0..7: acc0, 8..15: acc1
                if (lane < 16)
                    for (uint32_t i = lane; i < n16; i += 16) acc = __fmaf_rn(outv[i], outv[i], acc);
                const float other = __shfl_down_sync(0xffffffffu, acc, 8);  // acc1 lane l sits 8 lanes up
                const float both = __fadd_rn(acc, other);                   // lanes 0..7: acc0[l] + acc1[l]
                float sum = __shfl_sync(0xffffffffu, both, 0);
                for (int l = 1; l < 8; ++l) sum = __fadd_rn(sum, __shfl_sync(0xffffffffu, both, l));
                if (lane == 0) {
                    for (uint32_t i = n16; i < a.output_dim; ++i) sum = __fmaf_rn(outv[i], outv[i], sum);
                    s_scale = !(sum <= 0.0f);                                 // `if (sum <= 0.0f) return 0.0f;` leaves the vector as it is
                    s_inv = __fdiv_rn(1.0f, sqrtf(sum));
                }
            }
            __syncthreads();
            const float inv = s_inv;
            const bool scale_it = s_scale != 0;
            for (uint32_t row = threadIdx.x; row < a.output_dim; row += ENC_THREADS)
                a.out[(size_t)t * a.output_dim + row] = scale_it ? __fmul_rn(outv[row], inv) : outv[row];
        } else {
            for (uint32_t row = threadIdx.x; row < a.output_dim; row += ENC_THREADS) a.out[(size_t)t * a.output_dim + row] = outv[row];
        }
        __syncthreads();
    }
}

// The dynamic shared-memory limit is an attribute of the kernel, shared by every encoder and host thread of the process.  Set
// per call to the caller's own size, one thread could lower it between another thread's set and launch, and that launch
// would fail.  So it is raised once per device, to the largest layout any accepted configuration needs (sketch_dim 16384,
// output_dim 4096): the attribute permits that much, it reserves nothing -- each launch still asks for its own size.
constexpr size_t ENC_SMEM_MAX = (size_t)16384 * 4 * 2 + (size_t)4096 * 4 + 64;
constexpr int ENC_MAX_DEVICES = 64;

cudaError_t enc_allow_max_smem(int device) {
    static std::once_flag once[ENC_MAX_DEVICES];
    static cudaError_t rc[ENC_MAX_DEVICES];
    if (device < 0 || device >= ENC_MAX_DEVICES) return cudaErrorInvalidDevice;
    std::call_once(once[device], [device] {
        rc[device] = cudaFuncSetAttribute(simeon_encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ENC_SMEM_MAX);
    });
    return rc[device];
}

}  // namespace yb

using namespace yb;

struct yams_b200_encoder {
    DeviceCtx* dev = nullptr;
    yams_simeon_config cfg{};
    uint32_t words_per_col = 0;
    float scale = 0.f;
    DevBuf table;
    // Fwht
    uint32_t pad_n = 0;
    float fwht_scale = 0.f;
    DevBuf signs, sample;
    std::mutex mu;
};

extern "C" {

void yams_b200_simeon_default_config(yams_simeon_config* cfg) {
    if (!cfg) return;
    // simeon_v1_384_config (src/simeon.cpp:75-93)
    cfg->ngram_min = 3;
    cfg->ngram_max = 5;
    cfg->sketch_dim = 4096;
    cfg->output_dim = 384;
    cfg->hash_seed = 0xA5A5A5A5A5A5A5A5ULL;
    cfg->projection_seed = 0xDEADBEEFCAFEBABEULL;
    cfg->l2_normalize = 1;
    cfg->flags = 0;
}

void yams_b200_simeon_yams_config(yams_simeon_config* cfg, uint32_t embedding_dim) {
    if (!cfg) return;
    // resolveEncoder with an unconfigured [embeddings.simeon] (simeon_embedding_backend.cpp:118-135): parse_ngram_mode("") ->
    // CharAndWord (:18-29), parse_projection_mode("") -> Fwht (:31-46), n-grams 3..5, sketch 4096, output = embedding_dim
    yams_b200_simeon_default_config(cfg);
    cfg->output_dim = embedding_dim ? embedding_dim : 1024;   // EmbeddingConfig::embedding_dim default (embedding_generator.h:42)
    cfg->flags = YAMS_SIMEON_WORD_TOKENS | YAMS_SIMEON_PROJECTION_FWHT;
}

yams_status_t yams_b200_simeon_create(void* self, const yams_simeon_config* cfg_in, yams_b200_encoder** out) {
    YB_TRY
    (void)self;
    YB_ARG(out, "out is null");
    *out = nullptr;
    yams_simeon_config cfg;
    if (cfg_in) cfg = *cfg_in; else yams_b200_simeon_default_config(&cfg);
    YB_ARG(cfg.ngram_min >= 1 && cfg.ngram_min <= cfg.ngram_max && cfg.ngram_max <= 64, "ngram range must be 1 <= min <= max <= 64");
    YB_ARG(cfg.sketch_dim >= 1 && cfg.sketch_dim <= 16384, "sketch_dim must be in 1..16384");
    YB_ARG(cfg.output_dim >= 1 && cfg.output_dim <= 4096, "output_dim must be in 1..4096");
    YB_ARG((cfg.flags & ~(YAMS_SIMEON_WORD_TOKENS | YAMS_SIMEON_PROJECTION_FWHT)) == 0, "unknown encoder flags");
    const bool fwht = (cfg.flags & YAMS_SIMEON_PROJECTION_FWHT) != 0;
    uint32_t pad_n = 1;
    while (pad_n < cfg.sketch_dim) pad_n <<= 1;                                         // projection.cpp:72-80 next_pow2
    // projection.cpp:167-170: "Fwht requires output_dim <= next_pow2(sketch_dim)"
    YB_ARG(!fwht || cfg.output_dim <= pad_n, "Fwht requires output_dim <= next_pow2(sketch_dim)");
    DeviceCtx* dev = nullptr;
    yams_status_t rc = ensure_device(&dev);
    if (rc != YAMS_OK) return rc;
    std::unique_ptr<yams_b200_encoder> e(new (std::nothrow) yams_b200_encoder());
    if (!e) return YAMS_ERR_INTERNAL;
    e->dev = dev;
    e->cfg = cfg;
    e->words_per_col = (cfg.output_dim + 15) / 16;
    // projection.cpp:128-129: inv_scale_ = 1.0f / std::sqrt((float)output_dim); achlioptas_scale_ = std::sqrt(3.0f) * inv_scale_
    const float inv_scale = 1.0f / sqrtf((float)cfg.output_dim);
    e->scale = sqrtf(3.0f) * inv_scale;
    cudaError_t ce = cudaSuccess;
    if (fwht) {
        // projection.cpp:149-186, evaluated once on the host: the sign diagonal is one splitmix64 chain over i, the row sample a
        // partial Fisher-Yates over [0, pad_n) driven by a second chain -- both inherently sequential and tiny
        e->pad_n = pad_n;
        e->fwht_scale = 1.0f / sqrtf((float)cfg.output_dim);
        std::vector<float> signs(pad_n);
        uint64_t rng = sm64_mix(cfg.projection_seed ^ 0x9E3779B97F4A7C15ULL);
        for (uint32_t i = 0; i < pad_n; ++i) {
            rng = sm64_mix(rng + i);
            signs[i] = (rng & 1ULL) ? -1.0f : 1.0f;
        }
        std::vector<uint32_t> idx(pad_n);
        for (uint32_t i = 0; i < pad_n; ++i) idx[i] = i;
        uint64_t srng = sm64_mix(cfg.projection_seed ^ 0xBF58476D1CE4E5B9ULL);
        for (uint32_t i = 0; i < cfg.output_dim; ++i) {
            srng = sm64_mix(srng + i);
            const uint32_t pick = i + (uint32_t)(srng % (uint64_t)(pad_n - i));
            std::swap(idx[i], idx[pick]);
        }
        if ((rc = e->signs.reserve((size_t)pad_n * 4)) != YAMS_OK || (rc = e->sample.reserve((size_t)cfg.output_dim * 4)) != YAMS_OK) return rc;
        ce = cudaMemcpy(e->signs.p, signs.data(), (size_t)pad_n * 4, cudaMemcpyHostToDevice);
        if (ce == cudaSuccess) ce = cudaMemcpy(e->sample.p, idx.data(), (size_t)cfg.output_dim * 4, cudaMemcpyHostToDevice);
    } else {
    const size_t words = (size_t)cfg.sketch_dim * e->words_per_col;
    rc = e->table.reserve(words * 4);
    if (rc != YAMS_OK) return rc;
    achlioptas_table_kernel<<<(unsigned)((words + 255) / 256), 256>>>(cfg.sketch_dim, cfg.output_dim, cfg.projection_seed, e->words_per_col,
                                                                      e->table.as<uint32_t>());
    }
    if (ce == cudaSuccess) ce = cudaDeviceSynchronize();
    if (ce != cudaSuccess) {
        set_last_error("encoder table build failed: %s", cudaGetErrorString(ce));
        return YAMS_ERR_INTERNAL;
    }
    *out = e.release();
    return YAMS_OK;
    YB_CATCH
}

void yams_b200_simeon_destroy(yams_b200_encoder* e) { delete e; }

yams_status_t yams_b200_simeon_encode(yams_b200_encoder* e, const char* const* texts, const size_t* lens, size_t n, float* out) {
    YB_TRY
    YB_ARG(e, "encoder is null");
    if (n == 0) return YAMS_OK;
    YB_ARG(texts && lens && out, "null argument");
    YB_ARG(n < (1ull << 31), "too many texts");
    YB_BIND(e);
    OpWsLease lease;
    OpWs* w = lease.w;
    if (!w) return YAMS_ERR_INTERNAL;
    std::vector<uint64_t> offs(n + 1, 0);
    for (size_t i = 0; i < n; ++i) {
        YB_ARG(texts[i] || lens[i] == 0, "null text");
        offs[i + 1] = offs[i] + lens[i];
    }
    const uint64_t total = offs[n];
    const uint32_t D = e->cfg.output_dim;
    yams_status_t rc;
    if ((rc = w->d[0].reserve(total + 64)) != YAMS_OK) return rc;
    if ((rc = w->d[1].reserve((n + 1) * 8)) != YAMS_OK) return rc;
    if ((rc = w->d[2].reserve(n * (size_t)D * 4)) != YAMS_OK) return rc;
    if ((rc = w->h.reserve(std::max<uint64_t>(total, 64))) != YAMS_OK) return rc;
    uint8_t* hp = w->h.as<uint8_t>();
    for (size_t i = 0; i < n; ++i)
        if (lens[i]) memcpy(hp + offs[i], texts[i], lens[i]);
    cudaStream_t st = w->st;
    if (total) YB_CUDA(cudaMemcpyAsync(w->d[0].p, hp, total, cudaMemcpyHostToDevice, st));
    YB_CUDA(cudaMemcpyAsync(w->d[1].p, offs.data(), (n + 1) * 8, cudaMemcpyHostToDevice, st));
    EncArgs a{};
    a.text = w->d[0].as<uint8_t>();
    a.offsets = w->d[1].as<uint64_t>();
    a.n = (uint32_t)n;
    a.kmin = e->cfg.ngram_min; a.kmax = e->cfg.ngram_max;
    a.sketch_dim = e->cfg.sketch_dim; a.output_dim = D; a.words_per_col = e->words_per_col;
    a.h0 = gram_hash_h0(e->cfg.hash_seed);
    a.table = e->table.as<uint32_t>();
    a.scale = e->scale;
    a.l2_normalize = e->cfg.l2_normalize;
    a.out = w->d[2].as<float>();
    a.flags = (uint32_t)e->cfg.flags;
    a.pad_n = e->pad_n;
    a.signs = e->signs.as<float>();
    a.sample = e->sample.as<uint32_t>();
    a.fwht_scale = e->fwht_scale;
    const size_t smem = (size_t)e->cfg.sketch_dim * 4 + (size_t)std::max(e->cfg.sketch_dim, e->pad_n) * 4 + (size_t)D * 4 + 64;
    YB_CUDA(enc_allow_max_smem(e->dev->device));
    const unsigned grid = (unsigned)std::min<size_t>(n, (size_t)e->dev->sm_count * 8);
    simeon_encode_kernel<<<grid, ENC_THREADS, smem, st>>>(a);
    YB_CUDA(cudaGetLastError());
    YB_CUDA(cudaMemcpyAsync(out, w->d[2].p, n * (size_t)D * 4, cudaMemcpyDeviceToHost, st));
    YB_CUDA(cudaStreamSynchronize(st));
    return YAMS_OK;
    YB_CATCH
}

}  // extern "C"
