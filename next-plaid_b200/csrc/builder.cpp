// builder.cpp -- pb_create_index: MmapIndex::create_with_kmeans (index.rs:1392 -> kmeans.rs:261-422 ->
// index.rs:551-911) with every numeric step on the GPU and the reference's index directory as the result
// (file set of index.rs:394-525, SURVEY.md appendix B), so the reference -- or pb_index_load -- can open it.
//
//   1. compute_kmeans (kmeans.rs:273-419): sample docs, K = 2^floor(log2(16 sqrt(avg_doclen D))), at most
//      256 points per centroid, Lloyd iterations on the device (pb_kmeans_fit), L2-normalised centroids
//   2. prepare_codec_artifacts (index.rs:182-287): held-out rows from the end of a doc sample -> bucket cutoffs /
//      weights, avg_residual, cluster_threshold (pb_codec_train)
//   3. per chunk of `batch_size` docs (index.rs:289-371, :420-473): nearest-centroid codes + packed residuals
//      (pb_codec_encode_chunk: wgmma certified assignment), {i}.codes.npy, {i}.residuals.npy, doclens.{i}.json,
//      {i}.metadata.json
//   4. inverted file (index.rs:850-873): built on the device by pb_index_open (no ivf given), exported to
//      ivf.npy / ivf_lengths.npy; metadata.json, plan.json
// Sample membership (ChaCha8 shuffles in the reference) and the k-means iteration itself (fastkmeans-rs) are
// parity-unpinned (SURVEY 8c): this file uses its own splitmix64 shuffles.  Everything downstream of the centroids
// and the held-out sample is bit-identical to the oracle (tests/test_gpu_create_index.py).
#include "engine_internal.h"

#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <cmath>
#include <cerrno>
#include <cstdio>
#include <cstring>
#include <numeric>
#include <string>
#include <vector>

namespace {

uint64_t splitmix64(uint64_t &s) {
    uint64_t z = (s += 0x9e3779b97f4a7c15ull);
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}

// first `take` entries of a seeded Fisher-Yates shuffle of 0..n-1
std::vector<long long> shuffled_prefix(long long n, long long take, uint64_t seed) {
    std::vector<long long> p((size_t)n);
    std::iota(p.begin(), p.end(), 0ll);
    uint64_t s = seed;
    take = std::min(take, n);
    for (long long i = 0; i < take; ++i) {
        const long long j = i + (long long)(splitmix64(s) % (uint64_t)(n - i));
        std::swap(p[(size_t)i], p[(size_t)j]);
    }
    p.resize((size_t)take);
    return p;
}

// NPY v1.0, header padded so the payload starts on a 64-byte boundary (what numpy and mmap.rs:1177-1250 write)
pb_status write_npy(const std::string &path, const char *descr, const std::vector<long long> &shape, const void *data,
                    size_t bytes) {
    std::string dict = std::string("{'descr': '") + descr + "', 'fortran_order': False, 'shape': (";
    for (size_t i = 0; i < shape.size(); ++i) dict += std::to_string(shape[i]) + (shape.size() == 1 || i + 1 < shape.size() ? "," : "") + (i + 1 < shape.size() ? " " : "");
    dict += "), }";
    size_t total = 10 + dict.size() + 1;
    const size_t pad = (64 - total % 64) % 64;
    dict.append(pad, ' ');
    dict.push_back('\n');
    FILE *f = fopen(path.c_str(), "wb");
    if (!f) return pb_fail(PB_ERR_IO, "cannot create %s", path.c_str());
    const unsigned char magic[8] = {0x93, 'N', 'U', 'M', 'P', 'Y', 1, 0};
    const uint16_t hlen = (uint16_t)dict.size();
    bool ok = fwrite(magic, 1, 8, f) == 8 && fwrite(&hlen, 2, 1, f) == 1 && fwrite(dict.data(), 1, dict.size(), f) == dict.size();
    if (ok && bytes) ok = fwrite(data, 1, bytes, f) == bytes;
    ok = (fclose(f) == 0) && ok;
    return ok ? PB_OK : pb_fail(PB_ERR_IO, "short write to %s", path.c_str());
}

pb_status write_text(const std::string &path, const std::string &txt) {
    FILE *f = fopen(path.c_str(), "wb");
    if (!f) return pb_fail(PB_ERR_IO, "cannot create %s", path.c_str());
    bool ok = fwrite(txt.data(), 1, txt.size(), f) == txt.size();
    ok = (fclose(f) == 0) && ok;
    return ok ? PB_OK : pb_fail(PB_ERR_IO, "short write to %s", path.c_str());
}

// atomic_write_file (utils.rs:16-60): written and synced under a temporary name, then renamed over `path`
template <class Write> pb_status atomic_write(const std::string &path, Write write) {
    const std::string tmp = path + ".tmp";
    pb_status s = write(tmp);
    if (!s) {
        const int fd = open(tmp.c_str(), O_RDONLY);
        if (fd < 0 || fsync(fd) != 0) s = pb_fail(PB_ERR_IO, "cannot sync %s", tmp.c_str());
        if (fd >= 0) close(fd);
    }
    if (!s && rename(tmp.c_str(), path.c_str()) != 0) s = pb_fail(PB_ERR_IO, "cannot rename %s to %s", tmp.c_str(), path.c_str());
    if (s) remove(tmp.c_str());
    return s;
}

struct CodecGuard {
    pb_codec *c = nullptr;
    ~CodecGuard() {
        if (c) pb_codec_close(c);
    }
};

}  // namespace

extern "C" void pb_create_params_default(pb_create_params *p) {  // IndexConfig::default(), index.rs:88-102
    if (!p) return;
    p->nbits = 4;
    p->kmeans_niters = 4;
    p->max_points_per_centroid = 256;
    p->device = 0;
    p->num_partitions = 0;
    p->batch_size = 50000;
    p->seed = 42;
}

extern "C" pb_status pb_create_index(const float *embeddings, const int64_t *doc_lengths, int64_t n_docs, int32_t dim,
                                     const pb_create_params *params, const char *index_dir, pb_index **out_index) {
    if (!embeddings || !doc_lengths || !params || !index_dir) return pb_fail(PB_ERR_INVALID, "null argument");
    if (out_index) *out_index = nullptr;
    if (n_docs <= 0) return pb_fail(PB_ERR_INVALID, "no documents");
    const pb_create_params &cfg = *params;
    if (cfg.nbits <= 0 || 8 % cfg.nbits != 0) return pb_fail(PB_ERR_INVALID, "nbits must be a divisor of 8, got %d", cfg.nbits);
    if (cfg.batch_size <= 0 || cfg.kmeans_niters < 0 || cfg.max_points_per_centroid <= 0)
        return pb_fail(PB_ERR_INVALID, "bad create parameters");
    const long long D = n_docs;
    std::vector<long long> off((size_t)D + 1, 0);
    for (long long i = 0; i < D; ++i) {
        if (doc_lengths[i] < 0) return pb_fail(PB_ERR_INVALID, "doc_lengths[%lld] < 0", i);
        off[(size_t)i + 1] = off[(size_t)i] + doc_lengths[i];
    }
    const long long N = off[(size_t)D];
    if (N <= 0) return pb_fail(PB_ERR_INVALID, "no embeddings");
    mkdir(index_dir, 0777);
    const std::string dir = std::string(index_dir) + "/";
    const int packed = dim * cfg.nbits / 8;

    // ---- 1. centroids (kmeans.rs:273-419) ----
    const long long n_sdocs = pb_kmeans_num_sample_docs(D);
    const std::vector<long long> sdocs = shuffled_prefix(D, n_sdocs, cfg.seed);
    long long n_stok = 0;
    for (long long d : sdocs) n_stok += doc_lengths[d];
    if (n_stok <= 0) return pb_fail(PB_ERR_INVALID, "the k-means sample holds no embeddings");
    long long K = cfg.num_partitions > 0 ? std::min<long long>(cfg.num_partitions, n_stok)
                                         : pb_kmeans_num_partitions(D, (double)n_stok / (double)n_sdocs, n_stok);
    std::vector<float> samples((size_t)n_stok * dim);
    {
        size_t w = 0;
        for (long long d : sdocs) {
            const size_t n = (size_t)doc_lengths[d] * dim;
            memcpy(samples.data() + w, embeddings + (size_t)off[(size_t)d] * dim, n * sizeof(float));
            w += n;
        }
    }
    long long n_fit = n_stok;
    if (n_stok > K * (long long)cfg.max_points_per_centroid) {  // at most max_points_per_centroid points per centroid
        n_fit = K * (long long)cfg.max_points_per_centroid;
        const std::vector<long long> pick = shuffled_prefix(n_stok, n_fit, cfg.seed ^ 0x5bd1e995u);
        std::vector<float> sub((size_t)n_fit * dim);
        for (long long i = 0; i < n_fit; ++i)
            memcpy(sub.data() + (size_t)i * dim, samples.data() + (size_t)pick[(size_t)i] * dim, (size_t)dim * sizeof(float));
        samples.swap(sub);
    }
    std::vector<float> centroids((size_t)K * dim);
    if (pb_status s = pb_kmeans_fit(cfg.device, samples.data(), n_fit, dim, K, cfg.kmeans_niters, cfg.seed, centroids.data()))
        return s;
    std::vector<float>().swap(samples);

    // ---- 2. codec training on held-out rows (index.rs:195-287) ----
    CodecGuard cg;
    if (pb_status s = pb_codec_open(cfg.device, centroids.data(), K, dim, cfg.nbits, nullptr, &cg.c)) return s;
    const long long n_cdocs = pb_codec_num_sample_docs(D);
    const std::vector<long long> cdocs = shuffled_prefix(D, n_cdocs, cfg.seed + 1);
    const long long want = pb_codec_heldout_tokens(N);
    std::vector<float> heldout;
    long long got = 0;
    for (long long i = (long long)cdocs.size() - 1; i >= 0 && got < want; --i) {  // from the end of the sample list
        const long long d = cdocs[(size_t)i];
        const long long take = std::min<long long>(want - got, doc_lengths[d]);
        heldout.insert(heldout.end(), embeddings + (size_t)off[(size_t)d] * dim, embeddings + (size_t)(off[(size_t)d] + take) * dim);
        got += take;
    }
    const int nopt = 1 << cfg.nbits;
    std::vector<float> cutoffs((size_t)std::max(nopt - 1, 1)), weights((size_t)nopt), avg_res((size_t)dim);
    float threshold = 0.0f;
    if (pb_status s = pb_codec_train(cg.c, heldout.data(), got, cutoffs.data(), weights.data(), avg_res.data(), &threshold))
        return s;

    // ---- 3. encode chunk by chunk, write the chunk files (index.rs:420-473) ----
    std::vector<int64_t> codes((size_t)N);
    std::vector<uint8_t> residuals((size_t)N * packed);
    const long long n_chunks = (D + cfg.batch_size - 1) / cfg.batch_size;
    for (long long c = 0; c < n_chunks; ++c) {
        const long long d0 = c * cfg.batch_size, d1 = std::min<long long>(D, d0 + cfg.batch_size);
        const long long t0 = off[(size_t)d0], n = off[(size_t)d1] - t0;
        if (pb_status s = pb_codec_encode_chunk(cg.c, embeddings + (size_t)t0 * dim, n, codes.data() + t0,
                                                residuals.data() + (size_t)t0 * packed))
            return s;
        const std::string ci = std::to_string(c);
        if (pb_status s = write_npy(dir + ci + ".codes.npy", "<i8", {n}, codes.data() + t0, (size_t)n * 8)) return s;
        if (pb_status s = write_npy(dir + ci + ".residuals.npy", "|u1", {n, packed}, residuals.data() + (size_t)t0 * packed,
                                    (size_t)n * packed))
            return s;
        std::string dl = "[";
        for (long long d = d0; d < d1; ++d) dl += std::to_string((long long)doc_lengths[d]) + (d + 1 < d1 ? "," : "");
        dl += "]";
        if (pb_status s = write_text(dir + "doclens." + ci + ".json", dl)) return s;
        char meta[256];
        snprintf(meta, sizeof meta, "{\n  \"num_documents\": %lld,\n  \"num_embeddings\": %lld,\n  \"embedding_offset\": %lld\n}",
                 d1 - d0, n, t0);
        if (pb_status s = write_text(dir + ci + ".metadata.json", meta)) return s;
    }

    // ---- 4. inverted file on the device, remaining files ----
    pb_index_desc desc;
    memset(&desc, 0, sizeof desc);
    desc.dim = dim;
    desc.nbits = cfg.nbits;
    desc.num_centroids = K;
    desc.num_documents = D;
    desc.num_embeddings = N;
    desc.centroids = centroids.data();
    desc.bucket_weights = weights.data();
    desc.codes = codes.data();
    desc.residuals = residuals.data();
    desc.doc_lengths = doc_lengths;
    desc.device = cfg.device;
    desc.memory_space = PB_MEM_HOST;
    pb_index *ix = nullptr;
    if (pb_status s = pb_index_open(&desc, &ix)) return s;
    int64_t ivf_total = 0;
    pb_status st = pb_index_export_ivf(ix, nullptr, nullptr, &ivf_total);
    std::vector<int64_t> ivf((size_t)std::max<int64_t>(ivf_total, 1));
    std::vector<int32_t> ivf_len((size_t)K);
    if (!st) st = pb_index_export_ivf(ix, ivf.data(), ivf_len.data(), &ivf_total);
    if (!st) st = write_npy(dir + "ivf.npy", "<i8", {(long long)ivf_total}, ivf.data(), (size_t)ivf_total * 8);
    if (!st) st = write_npy(dir + "ivf_lengths.npy", "<i4", {K}, ivf_len.data(), (size_t)K * 4);
    if (!st) st = write_npy(dir + "centroids.npy", "<f4", {K, dim}, centroids.data(), (size_t)K * dim * 4);
    if (!st) st = write_npy(dir + "bucket_cutoffs.npy", "<f4", {(long long)nopt - 1}, cutoffs.data(), (size_t)(nopt - 1) * 4);
    if (!st) st = write_npy(dir + "bucket_weights.npy", "<f4", {(long long)nopt}, weights.data(), (size_t)nopt * 4);
    if (!st) st = write_npy(dir + "avg_residual.npy", "<f4", {(long long)dim}, avg_res.data(), (size_t)dim * 4);
    if (!st) st = write_npy(dir + "cluster_threshold.npy", "<f4", {1}, &threshold, 4);
    if (!st) {
        char plan[128];
        snprintf(plan, sizeof plan, "{\n  \"nbits\": %d,\n  \"num_chunks\": %lld\n}", cfg.nbits, n_chunks);
        st = write_text(dir + "plan.json", plan);
    }
    if (!st) {
        char meta[512];  // struct Metadata, index.rs:105-127
        snprintf(meta, sizeof meta,
                 "{\n  \"num_chunks\": %lld,\n  \"nbits\": %d,\n  \"num_partitions\": %lld,\n  \"num_embeddings\": %lld,\n"
                 "  \"avg_doclen\": %.17g,\n  \"num_documents\": %lld,\n  \"embedding_dim\": %d,\n  \"next_plaid_compatible\": true\n}",
                 n_chunks, cfg.nbits, K, N, (double)N / (double)D, D, dim);
        st = write_text(dir + "metadata.json", meta);
    }
    if (st || !out_index) pb_index_close(ix);
    else *out_index = ix;
    return st;
}

// Metadata::load_from_path (index.rs:131-155) of a directory that must hold the handle's old_D documents and nbits:
// num_documents 0 or absent is inferred from the doclens files
static pb_status read_dir_meta(const std::string &dir, int nbits, long long old_D, long long &num_chunks, long long &num_emb,
                               double &avg_doclen) {
    std::string meta;
    if (pb_status s = pb_read_text(dir + "metadata.json", meta)) return s;
    double nc = 0, mnbits = 0, ne = 0, num_docs = 0;
    if (!pb_json_number(meta, "num_chunks", nc) || !pb_json_number(meta, "nbits", mnbits) ||
        !pb_json_number(meta, "num_embeddings", ne) || !pb_json_number(meta, "avg_doclen", avg_doclen))
        return pb_fail(PB_ERR_IO, "metadata.json lacks num_chunks / nbits / num_embeddings / avg_doclen");
    num_chunks = (long long)nc;
    num_emb = (long long)ne;
    pb_json_number(meta, "num_documents", num_docs);
    long long meta_D = (long long)num_docs;
    if (meta_D == 0) {
        std::vector<int64_t> all;
        for (long long c = 0; c < num_chunks; ++c) pb_read_doclens(dir + "doclens." + std::to_string(c) + ".json", all);
        meta_D = (long long)all.size();
    }
    if ((int)mnbits != nbits) return pb_fail(PB_ERR_INVALID, "metadata.json nbits %d, the index has %d", (int)mnbits, nbits);
    if (meta_D != old_D)
        return pb_fail(PB_ERR_INVALID, "metadata.json num_documents %lld, the handle holds %lld documents", meta_D, old_D);
    return PB_OK;
}

pb_status pb_dir_check_documents(const char *index_dir, int nbits, long long D) {
    long long num_chunks = 0, num_emb = 0;
    double avg_doclen = 0;
    return read_dir_meta(std::string(index_dir) + "/", nbits, D, num_chunks, num_emb, avg_doclen);
}

// ivf.npy / ivf_lengths.npy
static pb_status write_ivf(const std::string &dir, long long K, const int64_t *ivf, long long ivf_total,
                           const int32_t *ivf_lengths) {
    pb_status s = atomic_write(dir + "ivf.npy", [&](const std::string &p) {
        return write_npy(p, "<i8", {ivf_total}, ivf, (size_t)ivf_total * 8);
    });
    if (!s) s = atomic_write(dir + "ivf_lengths.npy", [&](const std::string &p) {
        return write_npy(p, "<i4", {K}, ivf_lengths, (size_t)K * 4);
    });
    return s;
}

// metadata.json (struct Metadata, index.rs:105-127), then clear_merged_files (mmap.rs:1714-1740): the merged caches no
// longer match the chunks
static pb_status write_meta_clear_merged(const std::string &dir, long long num_chunks, int nbits, long long K, long long N,
                                         double avg_doclen, long long D, int dim) {
    char m[512];
    snprintf(m, sizeof m,
             "{\n  \"num_chunks\": %lld,\n  \"nbits\": %d,\n  \"num_partitions\": %lld,\n  \"num_embeddings\": %lld,\n"
             "  \"avg_doclen\": %.17g,\n  \"num_documents\": %lld,\n  \"embedding_dim\": %d,\n  \"next_plaid_compatible\": true\n}",
             num_chunks, nbits, K, N, avg_doclen, D, dim);
    if (pb_status s = atomic_write(dir + "metadata.json", [&](const std::string &p) { return write_text(p, m); })) return s;
    for (const char *f : {"merged_codes.npy", "merged_codes.npy.tmp", "merged_codes.manifest.json", "merged_codes.manifest.json.tmp",
                          "merged_residuals.npy", "merged_residuals.npy.tmp", "merged_residuals.manifest.json",
                          "merged_residuals.manifest.json.tmp"})
        if (remove((dir + f).c_str()) != 0 && errno != ENOENT) return pb_fail(PB_ERR_IO, "cannot remove %s%s", dir.c_str(), f);
    return PB_OK;
}

static std::string json_list(const std::vector<int64_t> &v) {
    std::string s = "[";
    for (size_t i = 0; i < v.size(); ++i) s += std::to_string((long long)v[i]) + (i + 1 < v.size() ? "," : "");
    return s + "]";
}

pb_status pb_dir_append(const char *index_dir, long long old_D, long long K, int dim, int nbits, long long batch_size,
                        const int64_t *codes, const uint8_t *residuals, const int64_t *doc_lengths, long long n_docs,
                        const int64_t *ivf, long long ivf_total, const int32_t *ivf_lengths) {
    const std::string dir = std::string(index_dir) + "/";
    const long long packed = (long long)dim * nbits / 8;
    long long n_chunks_old = 0, old_N = 0;
    double avg_doclen = 0;
    if (pb_status s = read_dir_meta(dir, nbits, old_D, n_chunks_old, old_N, avg_doclen)) return s;

    // a last chunk with < 2000 docs takes the first new batch (update.rs:799-827)
    long long start = n_chunks_old, emb_off = old_N;
    bool to_last = false;
    if (start > 0) {
        std::string lm;
        const std::string last = dir + std::to_string(start - 1) + ".metadata.json";
        double nd = 0, off = 0, ne = 0;
        if (access(last.c_str(), F_OK) == 0) {
            if (pb_status s = pb_read_text(last, lm)) return s;
            if (pb_json_number(lm, "num_documents", nd) && nd < 2000) {
                start -= 1;
                to_last = true;
                if (pb_json_number(lm, "embedding_offset", off)) emb_off = (long long)off;
                else emb_off = old_N - (pb_json_number(lm, "num_embeddings", ne) ? (long long)ne : 0);
            }
        }
    }
    const long long n_new_chunks = (n_docs + batch_size - 1) / batch_size;
    long long tok = 0;
    for (long long i = 0; i < n_new_chunks; ++i) {
        const std::string ci = std::to_string(start + i);
        const long long d0 = i * batch_size, d1 = std::min(n_docs, d0 + batch_size);
        std::vector<int64_t> cdl(doc_lengths + d0, doc_lengths + d1), ccodes;
        long long ntok = 0;
        for (int64_t v : cdl) ntok += v;
        ccodes.assign(codes + tok, codes + tok + ntok);
        std::vector<uint8_t> cres(residuals + (size_t)tok * packed, residuals + (size_t)(tok + ntok) * packed);
        tok += ntok;
        const std::string old_dl = dir + "doclens." + ci + ".json";
        if (i == 0 && to_last && access(old_dl.c_str(), F_OK) == 0) {  // prepend the old chunk, read from disk
            std::vector<int64_t> odl, ocodes;
            std::vector<uint8_t> ores;
            if (pb_status s = pb_read_doclens(old_dl, odl)) return s;
            long long otok = 0;
            for (int64_t v : odl) otok += v;
            if (pb_status s = pb_read_chunk(dir, start + i, otok, packed, ocodes, ores)) return s;
            cdl.insert(cdl.begin(), odl.begin(), odl.end());
            ccodes.insert(ccodes.begin(), ocodes.begin(), ocodes.end());
            cres.insert(cres.begin(), ores.begin(), ores.end());
        }
        const long long ctok = (long long)ccodes.size();
        pb_status s = atomic_write(dir + ci + ".codes.npy", [&](const std::string &p) {
            return write_npy(p, "<i8", {ctok}, ccodes.data(), (size_t)ctok * 8);
        });
        if (!s) s = atomic_write(dir + ci + ".residuals.npy", [&](const std::string &p) {
            return write_npy(p, "|u1", {ctok, packed}, cres.data(), cres.size());
        });
        const std::string dl = json_list(cdl);
        if (!s) s = atomic_write(old_dl, [&](const std::string &p) { return write_text(p, dl); });
        char cm[256];
        snprintf(cm, sizeof cm, "{\n  \"num_documents\": %lld,\n  \"num_embeddings\": %lld,\n  \"embedding_offset\": %lld\n}",
                 (long long)cdl.size(), ctok, emb_off);
        emb_off += ctok;
        if (!s) s = atomic_write(dir + ci + ".metadata.json", [&](const std::string &p) { return write_text(p, cm); });
        if (s) return s;
    }
    if (pb_status s = write_ivf(dir, K, ivf, ivf_total, ivf_lengths)) return s;
    // update.rs:1085-1110: avg_doclen from the file's old value, not N / D
    const long long total_D = old_D + n_docs;
    const double new_avg = total_D > 0 ? (avg_doclen * (double)old_D + (double)tok) / (double)total_D : 0.0;
    return write_meta_clear_merged(dir, start + n_new_chunks, nbits, K, old_N + tok, new_avg, total_D, dim);
}

// clean_embeddings_files (delete.rs:286-398) for one file pair: the rows of the documents that survive, doc i of the
// lengths file being doc id first + i; the files are removed when no document survives.  `info` (buffer_info.json) is
// rewritten or removed with them.
template <class Deleted>
static pb_status clean_embeddings_file(const std::string &dir, const char *npy, const char *lengths, const char *info,
                                       long long first_from_end, Deleted deleted) {
    const std::string ep = dir + npy, lp = dir + lengths;
    if (access(ep.c_str(), F_OK) != 0 || access(lp.c_str(), F_OK) != 0) return PB_OK;
    long long rows = 0, cols = 0;
    std::vector<float> flat, out;
    std::vector<int64_t> lens, kept;
    if (pb_status s = pb_read_npy_f32(ep, rows, cols, flat)) return s;
    if (pb_status s = pb_read_doclens(lp, lens)) return s;
    // embeddings.npy holds docs 0.., buffer.npy the last len(buffer_lengths) docs of the index before the delete
    const long long first = first_from_end < 0 ? 0 : first_from_end - (long long)lens.size();
    long long off = 0;
    for (size_t i = 0; i < lens.size(); ++i) {
        if (!deleted(first + (long long)i)) {
            for (long long r = off; r < off + lens[i] && r < rows; ++r) out.insert(out.end(), flat.begin() + r * cols, flat.begin() + (r + 1) * cols);
            kept.push_back(lens[i]);
        }
        off += lens[i];
    }
    if (kept.empty()) {
        remove(ep.c_str());
        remove(lp.c_str());
        if (info) remove((dir + info).c_str());
        return PB_OK;
    }
    const long long n_rows = cols ? (long long)out.size() / cols : 0;
    pb_status s = atomic_write(ep, [&](const std::string &p) { return write_npy(p, "<f4", {n_rows, cols}, out.data(), out.size() * 4); });
    const std::string lt = json_list(kept);
    if (!s) s = atomic_write(lp, [&](const std::string &p) { return write_text(p, lt); });
    const std::string it = "{\"num_docs\":" + std::to_string(kept.size()) + "}";
    if (!s && info) s = atomic_write(dir + info, [&](const std::string &p) { return write_text(p, it); });
    return s;
}

pb_status pb_dir_delete(const char *index_dir, long long old_D, long long K, int dim, int nbits, const uint32_t *deleted,
                        const int64_t *ivf, long long ivf_total, const int32_t *ivf_lengths) {
    const std::string dir = std::string(index_dir) + "/";
    const long long packed = (long long)dim * nbits / 8;
    long long n_chunks = 0, old_N = 0;
    double avg_doclen = 0;
    if (pb_status s = read_dir_meta(dir, nbits, old_D, n_chunks, old_N, avg_doclen)) return s;
    auto is_del = [&](long long d) { return d >= 0 && d < old_D && ((deleted[d >> 5] >> (d & 31)) & 1u); };
    // every chunk's doc lengths before the first write
    std::vector<std::vector<int64_t>> dls((size_t)n_chunks);
    long long total = 0;
    for (long long c = 0; c < n_chunks; ++c) {
        if (pb_status s = pb_read_doclens(dir + "doclens." + std::to_string(c) + ".json", dls[(size_t)c])) return s;
        total += (long long)dls[(size_t)c].size();
    }
    if (total != old_D)
        return pb_fail(PB_ERR_INVALID, "the doclens files hold %lld documents, the handle %lld", total, old_D);

    // per chunk (delete.rs:92-185): only chunks with a deleted doc are rewritten; num_chunks stays, embedding_offset too
    long long doc0 = 0, D1 = 0, N1 = 0;
    for (long long c = 0; c < n_chunks; ++c) {
        const std::vector<int64_t> &dl = dls[(size_t)c];
        std::vector<int64_t> ndl;
        long long ctok = 0;
        for (size_t i = 0; i < dl.size(); ++i) {
            ctok += dl[i];
            if (!is_del(doc0 + (long long)i)) {
                ndl.push_back(dl[i]);
                N1 += dl[i];
            }
        }
        D1 += (long long)ndl.size();
        if (ndl.size() < dl.size()) {
            const std::string ci = std::to_string(c);
            std::vector<int64_t> codes, ncodes;
            std::vector<uint8_t> res, nres;
            if (pb_status s = pb_read_chunk(dir, c, ctok, packed, codes, res)) return s;
            std::string cm;
            if (pb_status s = pb_read_text(dir + ci + ".metadata.json", cm)) return s;
            long long t = 0;
            for (size_t i = 0; i < dl.size(); ++i) {
                if (!is_del(doc0 + (long long)i)) {
                    ncodes.insert(ncodes.end(), codes.begin() + t, codes.begin() + t + dl[i]);
                    nres.insert(nres.end(), res.begin() + t * packed, res.begin() + (t + dl[i]) * packed);
                }
                t += dl[i];
            }
            const long long nt = (long long)ncodes.size();
            pb_status s = atomic_write(dir + ci + ".codes.npy", [&](const std::string &p) {
                return write_npy(p, "<i8", {nt}, ncodes.data(), (size_t)nt * 8);
            });
            if (!s) s = atomic_write(dir + ci + ".residuals.npy", [&](const std::string &p) {
                return write_npy(p, "|u1", {nt, packed}, nres.data(), nres.size());
            });
            const std::string dtxt = json_list(ndl);
            if (!s) s = atomic_write(dir + "doclens." + ci + ".json", [&](const std::string &p) { return write_text(p, dtxt); });
            double eo = 0;
            char m[256];
            if (pb_json_number(cm, "embedding_offset", eo))
                snprintf(m, sizeof m, "{\n  \"num_documents\": %lld,\n  \"num_embeddings\": %lld,\n  \"embedding_offset\": %lld\n}",
                         (long long)ndl.size(), nt, (long long)eo);
            else snprintf(m, sizeof m, "{\n  \"num_documents\": %lld,\n  \"num_embeddings\": %lld\n}", (long long)ndl.size(), nt);
            if (!s) s = atomic_write(dir + ci + ".metadata.json", [&](const std::string &p) { return write_text(p, m); });
            if (s) return s;
        }
        doc0 += (long long)dl.size();
    }
    if (pb_status s = write_ivf(dir, K, ivf, ivf_total, ivf_lengths)) return s;
    // delete.rs:240-260: avg_doclen = N / D of what is left (not the append's incremental formula)
    const double avg = D1 > 0 ? (double)N1 / (double)D1 : 0.0;
    if (pb_status s = write_meta_clear_merged(dir, n_chunks, nbits, K, N1, avg, D1, dim)) return s;
    if (pb_status s = clean_embeddings_file(dir, "embeddings.npy", "embeddings_lengths.json", nullptr, -1, is_del)) return s;
    return clean_embeddings_file(dir, "buffer.npy", "buffer_lengths.json", "buffer_info.json", old_D, is_del);
}
