/* pool_oracle.c -- CPU restatement of next-plaid-onnx's token pooling, for the tests and tools/bench_pool.py.
 *
 * pool_document_embeddings (lib.rs:1632-1643) -> pool_embeddings_hierarchical (lib.rs:2249-2317, protected_tokens 1)
 *   -> pdist_cosine (hierarchy.rs:599-653), linkage_ward (:128-284), fcluster_maxclust (:426-517).
 * Line by line, with the reference's (2n-1)^2 distance matrix and cluster ids; compiled with -ffp-contract=off so that
 * every multiply and add rounds separately, as in the reference.  OpenMP over documents, as rayon there.
 * Return codes: 0 ok; 2 a nearest-neighbour chain revisited a cluster (the reference never terminates there).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define INVALID_NN SIZE_MAX

/* hierarchy.rs:599-653, condensed upper triangle */
void po_pdist_cosine(const float *x, int64_t n, int32_t dim, double *out) {
    double *norms = malloc(sizeof(double) * (size_t)(n ? n : 1));
    for (int64_t i = 0; i < n; ++i) {
        double s = 0.0;
        for (int32_t k = 0; k < dim; ++k) {
            double v = (double)x[i * dim + k];
            s += v * v;
        }
        norms[i] = sqrt(s);
    }
    size_t c = 0;
    for (int64_t i = 0; i < n; ++i)
        for (int64_t j = i + 1; j < n; ++j) {
            double dot = 0.0;
            for (int32_t k = 0; k < dim; ++k) dot += (double)x[i * dim + k] * (double)x[j * dim + k];
            double cs = (norms[i] > 0.0 && norms[j] > 0.0) ? dot / (norms[i] * norms[j]) : 0.0;
            double d = 1.0 - cs;
            out[c++] = d < 0.0 ? 0.0 : (d > 2.0 ? 2.0 : d);
        }
    free(norms);
}

static void find_nn(size_t i, const size_t *act, size_t nact, const double *dsq, size_t T, size_t *nn, double *nd) {
    *nn = INVALID_NN;
    *nd = INFINITY;
    for (size_t p = 0; p < nact; ++p) {
        size_t j = act[p];
        if (j == i) continue;
        double v = dsq[i * T + j];
        if (v < *nd) {
            *nd = v;
            *nn = j;
        }
    }
}

/* linkage_ward (hierarchy.rs:128-259): the first max_merges rows (n - 1 for the whole dendrogram) into out [.][4] */
int po_ward_linkage(const double *dist, int64_t n64, int64_t max_merges, double *out) {
    size_t n = (size_t)n64;
    if (n <= 1) return 0;
    size_t T = 2 * n - 1;
    double *dsq = malloc(sizeof(double) * T * T);
    for (size_t e = 0; e < T * T; ++e) dsq[e] = INFINITY;
    for (size_t i = 0; i < n; ++i) {
        for (size_t j = i + 1; j < n; ++j) {
            double d = dist[n * i - (i * (i + 1)) / 2 + j - i - 1];
            double d2 = d * d;
            dsq[i * T + j] = d2;
            dsq[j * T + i] = d2;
        }
        dsq[i * T + i] = 0.0;
    }
    size_t *sizes = malloc(sizeof(size_t) * T), *act = malloc(sizeof(size_t) * T), *cnn = malloc(sizeof(size_t) * T);
    size_t *chain = malloc(sizeof(size_t) * T);
    double *cd = malloc(sizeof(double) * T);
    for (size_t i = 0; i < T; ++i) {
        sizes[i] = 1;
        cnn[i] = INVALID_NN;
        cd[i] = INFINITY;
    }
    size_t nact = n;
    for (size_t i = 0; i < n; ++i) act[i] = i;
    for (size_t i = 0; i < n; ++i) find_nn(i, act, nact, dsq, T, &cnn[i], &cd[i]);
    size_t next = n, clen = 0;
    int rc = 0;
    for (int64_t m = 0; m < max_merges && m < (int64_t)n - 1; ++m) {
        if (clen == 0) chain[clen++] = act[0];
        for (;;) {
            size_t cur = chain[clen - 1], nn;
            double nd;
            if (cnn[cur] != INVALID_NN) {
                nn = cnn[cur];
                nd = cd[cur];
            } else {
                find_nn(cur, act, nact, dsq, T, &nn, &nd);
                cnn[cur] = nn;
                cd[cur] = nd;
            }
            if (clen >= 2 && chain[clen - 2] == nn) {
                size_t a = chain[--clen], b = chain[--clen];
                size_t lo = a < b ? a : b, hi = a < b ? b : a;
                size_t na = sizes[a], nb = sizes[b], ns = na + nb;
                out[m * 4 + 0] = (double)lo;
                out[m * 4 + 1] = (double)hi;
                out[m * 4 + 2] = sqrt(nd);
                out[m * 4 + 3] = (double)ns;
                size_t w = 0;
                for (size_t p = 0; p < nact; ++p)
                    if (act[p] != a && act[p] != b) act[w++] = act[p];
                nact = w;
                sizes[next] = ns;
                double dab = nd;
                for (size_t p = 0; p < nact; ++p) {
                    size_t k = act[p], nk = sizes[k];
                    double dak = dsq[a * T + k], dbk = dsq[b * T + k];
                    double total = (double)(na + nb + nk);
                    double v = ((double)(na + nk) * dak + (double)(nb + nk) * dbk - (double)nk * dab) / total;
                    dsq[next * T + k] = v;
                    dsq[k * T + next] = v;
                    if (cnn[k] == a || cnn[k] == b) cnn[k] = INVALID_NN;
                }
                act[nact++] = next;
                find_nn(next, act, nact, dsq, T, &cnn[next], &cd[next]);
                ++next;
                break;
            }
            if (clen >= nact) { /* the chain would repeat a cluster: the reference loops forever */
                rc = 2;
                goto done;
            }
            chain[clen++] = nn;
        }
    }
done:
    free(dsq);
    free(sizes);
    free(act);
    free(cnn);
    free(chain);
    free(cd);
    return rc;
}

static size_t uf_find(size_t *parent, size_t i) {
    while (parent[i] != i) i = parent[i];
    return i;
}

static size_t obs_in_cluster(const double *L, size_t n, size_t c) {
    while (c >= n) c = (size_t)L[(c - n) * 4 + 0];
    return c;
}

/* fcluster_maxclust (hierarchy.rs:426-504): labels 1.. numbered by first observation */
static void fcluster_maxclust(const double *L, size_t n, size_t maxc, size_t *labels) {
    if (maxc >= n) {
        for (size_t i = 0; i < n; ++i) labels[i] = i + 1;
        return;
    }
    if (maxc == 0) {
        for (size_t i = 0; i < n; ++i) labels[i] = 1;
        return;
    }
    size_t *parent = malloc(sizeof(size_t) * n), *rank = calloc(n, sizeof(size_t)), *map = malloc(sizeof(size_t) * n);
    for (size_t i = 0; i < n; ++i) {
        parent[i] = i;
        map[i] = 0;
    }
    for (size_t i = 0; i < n - maxc; ++i) {
        size_t c1 = (size_t)L[i * 4], c2 = (size_t)L[i * 4 + 1];
        size_t o1 = obs_in_cluster(L, n, c1), o2 = obs_in_cluster(L, n, c2);
        size_t p1 = uf_find(parent, o1), p2 = uf_find(parent, o2);
        if (p1 == p2) continue;
        if (rank[p1] < rank[p2]) parent[p1] = p2;
        else if (rank[p1] > rank[p2]) parent[p2] = p1;
        else {
            parent[p2] = p1;
            rank[p1] += 1;
        }
    }
    size_t next = 1;
    for (size_t i = 0; i < n; ++i) {
        size_t r = uf_find(parent, i);
        if (!map[r]) map[r] = next++;
        labels[i] = map[r];
    }
    free(parent);
    free(rank);
    free(map);
}

/* pool_embeddings_hierarchical(doc, pool_factor, 1) for one document of n rows into out; returns the row count, or
 * -2 when the chain does not terminate */
static int64_t pool_one(const float *x, int64_t n, int32_t dim, int64_t pf, float *out) {
    if (pf <= 1 || n <= 2) {
        memcpy(out, x, sizeof(float) * (size_t)n * dim);
        return n;
    }
    size_t t = (size_t)n - 1, k = t / (size_t)pf;
    if (k < 1) k = 1;
    if (k >= t) {
        memcpy(out, x, sizeof(float) * (size_t)n * dim);
        return n;
    }
    const float *tp = x + dim;
    double *dist = malloc(sizeof(double) * (t * (t - 1) / 2 + 1));
    double *L = malloc(sizeof(double) * 4 * t);
    size_t *labels = malloc(sizeof(size_t) * t);
    po_pdist_cosine(tp, (int64_t)t, dim, dist);
    int rc = po_ward_linkage(dist, (int64_t)t, (int64_t)(t - k), L);
    if (rc == 0) {
        fcluster_maxclust(L, t, k, labels);
        float *sums = calloc(k * (size_t)dim, sizeof(float));
        size_t *counts = calloc(k, sizeof(size_t));
        for (size_t i = 0; i < t; ++i) {
            size_t c = labels[i] - 1;
            if (c >= k) continue;
            for (int32_t f = 0; f < dim; ++f) sums[c * dim + f] += tp[i * dim + f];
            counts[c] += 1;
        }
        memcpy(out, x, sizeof(float) * dim);
        for (size_t c = 0; c < k; ++c) {
            float cnt = (float)(counts[c] ? counts[c] : 1);
            for (int32_t f = 0; f < dim; ++f) out[(1 + c) * dim + f] = sums[c * dim + f] / cnt;
        }
        free(sums);
        free(counts);
    }
    free(dist);
    free(L);
    free(labels);
    return rc ? -2 : (int64_t)(1 + k);
}

int64_t po_pooled_doc_length(int64_t n, int64_t pf) {
    if (pf <= 1 || n <= 2) return n;
    int64_t t = n - 1, k = t / pf;
    if (k < 1) k = 1;
    return k >= t ? n : 1 + k;
}

/* pool_document_embeddings over n_docs concatenated documents; out sized by po_pooled_doc_length */
int po_pool_embeddings(const float *x, const int64_t *lens, int64_t n_docs, int32_t dim, int64_t pf, float *out,
                       int64_t *out_lens) {
    int64_t *in_off = malloc(sizeof(int64_t) * (size_t)(n_docs + 1)), *out_off = malloc(sizeof(int64_t) * (size_t)(n_docs + 1));
    in_off[0] = out_off[0] = 0;
    for (int64_t i = 0; i < n_docs; ++i) {
        in_off[i + 1] = in_off[i] + lens[i];
        out_off[i + 1] = out_off[i] + po_pooled_doc_length(lens[i], pf);
    }
    int rc = 0;
#pragma omp parallel for schedule(dynamic, 4)
    for (int64_t i = 0; i < n_docs; ++i) {
        int64_t r = pool_one(x + in_off[i] * dim, lens[i], dim, pf, out + out_off[i] * dim);
        out_lens[i] = r;
        if (r < 0) {
#pragma omp atomic write
            rc = 2;
        }
    }
    free(in_off);
    free(out_off);
    return rc;
}
