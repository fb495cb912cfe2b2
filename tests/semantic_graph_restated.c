/* semantic_graph_restated.c -- plain-C restatement of the semantic-neighbour graph that YAMS's daemon builds over document-level
 * embeddings (EmbeddingService::updateSemanticNeighborGraphUnlocked, src/daemon/components/EmbeddingService.cpp).  It is the
 * oracle of yams_b200_semantic_neighbors: the daemon needs Boost and nlohmann_json and is not built as a test dependency.
 *
 * The corpus is rows[n][d] in document_hash order (one record per hash, :864-882), so row order is hash order.  Restated:
 *   inverseNorm        :405-415   sequential double sum of squares, 0 when <= 0, float(1 / sqrt)
 *   cosineSimilarity   :417-431   float((dot * (double)invA) * (double)invB), dot the sequential double sum, source first
 *   corpus filter      :875-877   rows with inv <= 0 are not in the corpus
 *   sources            :899-922   all corpus rows, or the requested ones that are in the corpus with inv > 0
 *   pair loop          :945-1011  own hash skipped; explicit threshold: sim < t dropped; adaptive: sim <= 0 dropped;
 *                                 replace-worst top-k under isBetterNeighbor (:934-942), sim desc then hash asc
 *   final sort         :1017      std::sort by isBetterNeighbor
 * The one rule the reference leaves undefined: a NaN similarity (a row with a NaN element has inv NaN and enters its corpus;
 * a row whose inv overflows to +inf scores 0 * inf = NaN where dot == 0) enters the top-k, which replace-worst and sort cannot
 * order.  Here a NaN similarity is never a neighbour, as in yams_b200_semantic_neighbors; a row with inv NaN is not a source
 * (inv > 0 fails, :904, 916).  Rows with inv = +inf are taken, with their +-inf similarities.
 * Build: cc -O2 -fopenmp -fPIC -shared (no -ffast-math: the sums must stay sequential). */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

static float inverse_norm(const float* v, uint32_t d) {
    double norm = 0.0;
    for (uint32_t i = 0; i < d; ++i) {
        const double xd = v[i];
        norm += xd * xd;
    }
    if (norm <= 0.0) return 0.0f;
    return (float)(1.0 / sqrt(norm));
}

static float cosine_similarity(const float* a, float inv_a, const float* b, float inv_b, uint32_t d) {
    if (inv_a <= 0.0f || inv_b <= 0.0f) return 0.0f;
    double dot = 0.0;
    for (uint32_t i = 0; i < d; ++i) dot += (double)a[i] * (double)b[i];
    return (float)(dot * inv_a * inv_b);
}

typedef struct {
    int64_t row;
    float sim;
} neighbor_t;

/* isBetterNeighbor (:934-939): hash ascending is row ascending */
static int is_better(const neighbor_t* l, const neighbor_t* r) {
    if (l->sim != r->sim) return l->sim > r->sim;
    return l->row < r->row;
}

static int cmp_better(const void* a, const void* b) {
    const neighbor_t* l = (const neighbor_t*)a;
    const neighbor_t* r = (const neighbor_t*)b;
    if (is_better(l, r)) return -1;
    if (is_better(r, l)) return 1;
    return 0;
}

/* the row is in the corpus and can be a source: inv > 0 (:875-877, :904, 916); NaN fails, +inf passes */
static int taken(float inv) { return inv > 0.0f; }

/* rows[n][d]; sources: NULL = every row, else n_src row indices (>= n: not in the corpus -> count 0).
 * adaptive != 0: no explicit threshold (sim <= 0 dropped), else sim < threshold dropped.
 * out_rows / out_sims [n_src][k] (unused: -1 / 0), out_counts[n_src].  inv_out (nullable) [n] receives inverseNorm of each row. */
int sg_semantic_neighbors(const float* rows, uint64_t n, uint32_t d, const int64_t* sources, uint64_t n_src, uint32_t k, int adaptive,
                          float threshold, int64_t* out_rows, float* out_sims, uint32_t* out_counts, float* inv_out) {
    float* inv = (float*)malloc((n ? n : 1) * sizeof(float));
    if (!inv) return -1;
    for (uint64_t r = 0; r < n; ++r) inv[r] = inverse_norm(rows + r * d, d);
    if (inv_out)
        for (uint64_t r = 0; r < n; ++r) inv_out[r] = inv[r];
    int failed = 0;
#pragma omp parallel for schedule(dynamic, 1)
    for (uint64_t i = 0; i < n_src; ++i) {
        for (uint32_t j = 0; j < k; ++j) {
            out_rows[i * k + j] = -1;
            out_sims[i * k + j] = 0.0f;
        }
        out_counts[i] = 0;
        const int64_t s = sources ? sources[i] : (int64_t)i;
        if (s < 0 || (uint64_t)s >= n || !taken(inv[s]) || k == 0) continue;
        neighbor_t* top = (neighbor_t*)malloc((size_t)k * sizeof(neighbor_t));
        if (!top) {
            failed = 1;
            continue;
        }
        uint32_t size = 0;
        for (uint64_t r = 0; r < n; ++r) {
            if ((int64_t)r == s || !taken(inv[r])) continue;
            const float sim = cosine_similarity(rows + (uint64_t)s * d, inv[s], rows + r * d, inv[r], d);
            if (sim != sim) continue; /* no reference answer (see above) */
            if (!adaptive) {
                if (sim < threshold) continue;
            } else if (sim <= 0.0f) {
                continue;
            }
            const neighbor_t cand = {(int64_t)r, sim};
            if (size < k) {
                top[size++] = cand;
                continue;
            }
            /* std::min_element under isWorseNeighbor: the first element no other is worse than */
            uint32_t worst = 0;
            for (uint32_t j = 1; j < size; ++j)
                if (is_better(&top[worst], &top[j])) worst = j;
            if (is_better(&cand, &top[worst])) top[worst] = cand;
        }
        qsort(top, size, sizeof(neighbor_t), cmp_better);
        for (uint32_t j = 0; j < size; ++j) {
            out_rows[i * k + j] = top[j].row;
            out_sims[i * k + j] = top[j].sim;
        }
        out_counts[i] = size;
        free(top);
    }
    free(inv);
    return failed ? -1 : 0;
}
