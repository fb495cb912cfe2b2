/* topology_kmeans_restated.c -- plain-C restatement of the k-means topology engine's clustering (KMeansTopologyEngine's
 * runKMeans, src/topology/topology_alternate_engines.cpp:288-478, meanEmbedding topology_build_utils.h:27-56).  It is the
 * oracle of yams_b200_topology_kmeans at sizes where the Python transcription (topology_kmeans_restated.py) is too slow.
 *
 * The input is the usable documents only, rows[n][d] in document order (the caller keeps the singletons).  Restated:
 *   cosineDistance     :288-305   dot, na, nb sequential double sums; 2.0 when na <= 0 || nb <= 0; 1 - clamp(cos, -1, 1), NaN kept
 *   normalized         :307-319   double sum of squares, inv = float(1 / sqrt), float multiply; unchanged when the sum <= 0
 *   nearestCentroid    :321-336   first centroid with the strictly smallest distance, 0 by default
 *   k                  :367-371   requested, or round(sqrt(n)) when 0, clamped to [2, n]
 *   init               :373-401   farthest-first, minDist strict <, first largest strict >
 *   iterations         :403-466   assignment, centroids of non-empty clusters, empty-cluster repairs in c order, stop when
 *                                 nothing changed; meanEmbedding's float sums from +0 in member order, / float(count)
 * OpenMP runs the loops over documents; every per-document value is computed in the reference's order, and the (max, first
 * index) reductions are done sequentially.
 * Build: cc -O2 -fopenmp -fPIC -shared (no -ffast-math: the sums must stay sequential). */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static double sumsq(const float* a, uint32_t d) {
    double s = 0.0;
    for (uint32_t i = 0; i < d; ++i) s += (double)a[i] * (double)a[i];
    return s;
}

static double cosine_distance(const float* a, const float* b, uint32_t d) {
    double dot = 0.0, na = 0.0, nb = 0.0;
    for (uint32_t i = 0; i < d; ++i) {
        dot += (double)a[i] * (double)b[i];
        na += (double)a[i] * (double)a[i];
        nb += (double)b[i] * (double)b[i];
    }
    if (na <= 0.0 || nb <= 0.0) return 2.0;
    const double cs = dot / (sqrt(na) * sqrt(nb));
    return 1.0 - (cs < -1.0 ? -1.0 : (1.0 < cs ? 1.0 : cs));
}

static void normalize_into(const float* v, uint32_t d, float* out) {
    const double norm = sumsq(v, d);
    if (norm > 0.0) {
        const float inv = (float)(1.0 / sqrt(norm));
        for (uint32_t i = 0; i < d; ++i) out[i] = v[i] * inv;
    } else {
        memmove(out, v, (size_t)d * sizeof(float));
    }
}

/* centroidOf: normalized(meanEmbedding(members)) of the members u (membership[u] == c) in u order; tmp holds d floats */
static void centroid_of(const float* rows, uint32_t n, uint32_t d, const uint32_t* membership, uint32_t c, float* tmp, float* out) {
    uint64_t count = 0;
    for (uint32_t i = 0; i < d; ++i) tmp[i] = 0.0f;
    for (uint32_t u = 0; u < n; ++u) {
        if (membership[u] != c) continue;
        const float* r = rows + (uint64_t)u * d;
        for (uint32_t i = 0; i < d; ++i) tmp[i] += r[i];
        ++count;
    }
    for (uint32_t i = 0; i < d; ++i) tmp[i] /= (float)count;
    normalize_into(tmp, d, out);
}

/* -> 0; out_assignment[n], out_centroids[k][d] (k <= k_cap, nullable), *out_k, *out_iterations.  n < 2: iota, k = 0. */
int tk_kmeans(const float* rows, uint32_t n, uint32_t d, uint32_t k_requested, uint32_t max_iterations, uint32_t* out_assignment,
              float* out_centroids, uint32_t* out_k, uint32_t* out_iterations) {
    *out_k = 0;
    *out_iterations = 0;
    if (n < 2) {
        for (uint32_t i = 0; i < n; ++i) out_assignment[i] = i;
        return 0;
    }
    uint64_t k = k_requested ? k_requested : (uint64_t)llround(sqrt((double)n));
    if (k < 2) k = 2;
    if (k > n) k = n;
    float* cent = malloc((size_t)k * d * sizeof(float));
    double* min_dist = malloc((size_t)n * sizeof(double));
    double* dist = malloc((size_t)n * sizeof(double));
    unsigned char* selected = calloc(n, 1);
    uint32_t* membership = calloc(n, sizeof(uint32_t));
    uint32_t* next = malloc((size_t)n * sizeof(uint32_t));
    uint64_t* size = malloc((size_t)k * sizeof(uint64_t));
    float* tmp = malloc((size_t)d * sizeof(float));

    normalize_into(rows, d, cent);
    selected[0] = 1;
    for (uint32_t u = 0; u < n; ++u) min_dist[u] = DBL_MAX;
    for (uint64_t s = 1; s < k; ++s) {
        const float* last = cent + (s - 1) * d;
#pragma omp parallel for schedule(static)
        for (uint32_t u = 0; u < n; ++u) {
            if (selected[u]) continue;
            const double dd = cosine_distance(rows + (uint64_t)u * d, last, d);
            if (dd < min_dist[u]) min_dist[u] = dd;
        }
        uint32_t far = n;
        double far_dist = -1.0;
        for (uint32_t u = 0; u < n; ++u)
            if (!selected[u] && min_dist[u] > far_dist) { far_dist = min_dist[u]; far = u; }
        if (far == n) break;   /* unreachable with k <= n, kept as the reference has it */
        selected[far] = 1;
        normalize_into(rows + (uint64_t)far * d, d, cent + s * d);
    }

    const uint32_t iterations = max_iterations == 0 ? 10 : max_iterations;
    uint32_t iter = 0;
    while (iter < iterations) {
        ++iter;
        int changed = 0;
#pragma omp parallel for schedule(static)
        for (uint32_t u = 0; u < n; ++u) {
            uint32_t best = 0;
            double best_dist = DBL_MAX;
            for (uint64_t c = 0; c < k; ++c) {
                const double dd = cosine_distance(rows + (uint64_t)u * d, cent + c * d, d);
                if (dd < best_dist) { best_dist = dd; best = (uint32_t)c; }
            }
            next[u] = best;
        }
        for (uint32_t u = 0; u < n; ++u) {
            if (next[u] != membership[u]) { membership[u] = next[u]; changed = 1; }
        }
        for (uint64_t c = 0; c < k; ++c) size[c] = 0;
        for (uint32_t u = 0; u < n; ++u) ++size[membership[u]];
        for (uint64_t c = 0; c < k; ++c)
            if (size[c]) centroid_of(rows, n, d, membership, (uint32_t)c, tmp, cent + c * d);
        for (uint64_t c = 0; c < k; ++c) {
            if (size[c]) continue;
#pragma omp parallel for schedule(static)
            for (uint32_t u = 0; u < n; ++u) {
                const uint32_t mc = membership[u];
                dist[u] = size[mc] <= 1 ? NAN : cosine_distance(rows + (uint64_t)u * d, cent + (uint64_t)mc * d, d);
            }
            uint32_t worst = n;
            double worst_dist = -1.0;
            for (uint32_t u = 0; u < n; ++u)
                if (dist[u] > worst_dist) { worst_dist = dist[u]; worst = u; }
            if (worst == n) continue;
            const uint32_t donor = membership[worst];
            membership[worst] = (uint32_t)c;
            size[donor] -= 1;
            size[c] = 1;
            normalize_into(rows + (uint64_t)worst * d, d, cent + c * d);
            centroid_of(rows, n, d, membership, donor, tmp, cent + (uint64_t)donor * d);
            changed = 1;
        }
        if (!changed) break;
    }
    memcpy(out_assignment, membership, (size_t)n * sizeof(uint32_t));
    if (out_centroids) memcpy(out_centroids, cent, (size_t)k * d * sizeof(float));
    *out_k = (uint32_t)k;
    *out_iterations = iter;
    free(cent); free(min_dist); free(dist); free(selected); free(membership); free(next); free(size); free(tmp);
    return 0;
}
