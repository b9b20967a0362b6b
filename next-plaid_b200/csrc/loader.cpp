// loader.cpp -- pb_index_load: MmapIndex::load (index.rs:1026-1139) for the GPU engine.
//
// Reads the reference's index directory as-is (SURVEY.md appendix B): metadata.json,
// centroids.npy, bucket_weights.npy, ivf.npy, ivf_lengths.npy, doclens.{i}.json and the chunk files
// {i}.codes.npy / {i}.residuals.npy, and uploads chunk by chunk so the host never holds the whole
// corpus.  The derived caches merged_codes.npy / merged_residuals.npy (mmap.rs:1266,1483) are not
// needed: their only extra content is the zero padding rows of index.rs:1113-1120.
// fast-plaid directories (f16 tensors, i64 ivf_lengths, mmap.rs:1757-1811) load too: widened / narrowed in memory.
#include "engine_internal.h"

#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <cctype>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

namespace {

struct Mapped {
    void *base = nullptr;
    size_t size = 0;
    ~Mapped() {
        if (base && base != MAP_FAILED) munmap(base, size);
    }
    pb_status open(const std::string &path) {
        int fd = ::open(path.c_str(), O_RDONLY);
        if (fd < 0) return pb_fail(PB_ERR_IO, "cannot open %s", path.c_str());
        struct stat st;
        if (fstat(fd, &st) != 0) {
            ::close(fd);
            return pb_fail(PB_ERR_IO, "cannot stat %s", path.c_str());
        }
        size = (size_t)st.st_size;
        if (size == 0) {
            ::close(fd);
            return pb_fail(PB_ERR_IO, "%s is empty", path.c_str());
        }
        base = mmap(nullptr, size, PROT_READ, MAP_PRIVATE, fd, 0);
        ::close(fd);
        if (base == MAP_FAILED) {
            base = nullptr;
            return pb_fail(PB_ERR_IO, "cannot mmap %s", path.c_str());
        }
        return PB_OK;
    }
};

// NPY v1/v2/v3 (mmap.rs:754-1010 reads the same header)
struct Npy {
    Mapped m;
    std::string descr;
    std::vector<long long> shape;
    const unsigned char *data = nullptr;
    size_t itemsize = 0;

    pb_status open(const std::string &path) {
        if (pb_status s = m.open(path)) return s;
        const unsigned char *p = (const unsigned char *)m.base;
        if (m.size < 12 || memcmp(p, "\x93NUMPY", 6) != 0) return pb_fail(PB_ERR_IO, "%s is not an NPY file", path.c_str());
        int major = p[6];
        size_t hlen, hoff;
        if (major == 1) {
            hlen = p[8] | (p[9] << 8);
            hoff = 10;
        } else {
            hlen = p[8] | (p[9] << 8) | (p[10] << 16) | ((size_t)p[11] << 24);
            hoff = 12;
        }
        if (hoff + hlen > m.size) return pb_fail(PB_ERR_IO, "%s: truncated NPY header", path.c_str());
        std::string h((const char *)p + hoff, hlen);
        size_t d = h.find("'descr'");
        if (d == std::string::npos) return pb_fail(PB_ERR_IO, "%s: NPY header has no descr", path.c_str());
        size_t q1 = h.find('\'', h.find(':', d));
        size_t q2 = h.find('\'', q1 + 1);
        if (q1 == std::string::npos || q2 == std::string::npos) return pb_fail(PB_ERR_IO, "%s: bad descr", path.c_str());
        descr = h.substr(q1 + 1, q2 - q1 - 1);
        size_t f = h.find("'fortran_order'");
        if (f != std::string::npos && h.compare(h.find(':', f) + 1, 5, " True") == 0)
            return pb_fail(PB_ERR_UNSUPPORTED, "%s: fortran_order arrays are not supported", path.c_str());
        size_t s = h.find("'shape'");
        size_t p1 = h.find('(', s), p2 = h.find(')', p1);
        if (s == std::string::npos || p1 == std::string::npos || p2 == std::string::npos)
            return pb_fail(PB_ERR_IO, "%s: bad shape", path.c_str());
        shape.clear();
        const char *c = h.c_str() + p1 + 1, *end = h.c_str() + p2;
        while (c < end) {
            while (c < end && !isdigit((unsigned char)*c)) ++c;
            if (c >= end) break;
            shape.push_back(strtoll(c, (char **)&c, 10));
        }
        itemsize = (size_t)atoi(descr.c_str() + 2);
        if (itemsize == 0) return pb_fail(PB_ERR_IO, "%s: bad descr %s", path.c_str(), descr.c_str());
        data = p + hoff + hlen;
        size_t n = 1;
        for (long long v : shape) n *= (size_t)v;
        if (hoff + hlen + n * itemsize > m.size) return pb_fail(PB_ERR_IO, "%s: truncated NPY payload", path.c_str());
        return PB_OK;
    }
    long long count() const {
        long long n = 1;
        for (long long v : shape) n *= v;
        return n;
    }
    bool is(const char *kind_size) const {  // e.g. "f4", "i8", "u1"
        return descr.size() >= 3 && descr.compare(1, 2, kind_size) == 0 && (descr[0] == '<' || descr[0] == '|' || descr[0] == '=');
    }
};

// IEEE half -> float (fast-plaid directories store their float tensors as <f2, mmap.rs:1757-1811)
float half_to_float(uint16_t h) {
    const uint32_t sign = (uint32_t)(h & 0x8000u) << 16, exp = (h >> 10) & 31u, man = h & 1023u;
    uint32_t bits;
    if (exp == 0) {
        if (man == 0) bits = sign;
        else {  // subnormal: renormalise
            int e = -1;
            uint32_t m = man;
            do {
                ++e;
                m <<= 1;
            } while (!(m & 1024u));
            bits = sign | ((uint32_t)(127 - 15 - e) << 23) | ((m & 1023u) << 13);
        }
    } else if (exp == 31) bits = sign | 0x7f800000u | (man << 13);
    else bits = sign | ((exp - 15 + 127) << 23) | (man << 13);
    float f;
    memcpy(&f, &bits, 4);
    return f;
}

// a float tensor of the directory as f32: <f4 is used in place, <f2 (fast-plaid) is widened into `store`
pb_status as_f32(const Npy &a, const char *name, std::vector<float> &store, const float **out) {
    if (a.is("f4")) {
        *out = (const float *)a.data;
        return PB_OK;
    }
    if (!a.is("f2")) return pb_fail(PB_ERR_IO, "%s must be <f4 (next-plaid) or <f2 (fast-plaid)", name);
    const long long n = a.count();
    store.resize((size_t)n);
    const uint16_t *src = (const uint16_t *)a.data;
    for (long long i = 0; i < n; ++i) store[(size_t)i] = half_to_float(src[i]);
    *out = store.data();
    return PB_OK;
}

}  // namespace

pb_status pb_read_text(const std::string &path, std::string &out) {
    FILE *f = fopen(path.c_str(), "rb");
    if (!f) return pb_fail(PB_ERR_IO, "cannot open %s", path.c_str());
    char buf[1 << 16];
    size_t n;
    out.clear();
    while ((n = fread(buf, 1, sizeof buf, f)) > 0) out.append(buf, n);
    fclose(f);
    return PB_OK;
}

// number following "key": in a flat JSON object (metadata.json, index.rs:105-127)
bool pb_json_number(const std::string &j, const char *key, double &out) {
    std::string k = std::string("\"") + key + "\"";
    size_t p = j.find(k);
    if (p == std::string::npos) return false;
    p = j.find(':', p + k.size());
    if (p == std::string::npos) return false;
    ++p;
    while (p < j.size() && isspace((unsigned char)j[p])) ++p;
    char *end = nullptr;
    out = strtod(j.c_str() + p, &end);
    return end != j.c_str() + p;
}

pb_status pb_read_doclens(const std::string &path, std::vector<int64_t> &out) {
    std::string txt;
    if (pb_status s = pb_read_text(path, txt)) return s;
    const char *p = txt.c_str();
    while (*p) {
        if (isdigit((unsigned char)*p) || (*p == '-' && isdigit((unsigned char)p[1]))) out.push_back(strtoll(p, (char **)&p, 10));
        else ++p;
    }
    return PB_OK;
}

pb_status pb_read_chunk(const std::string &dir, long long chunk, long long n_tokens, long long packed,
                        std::vector<int64_t> &codes, std::vector<uint8_t> &residuals) {
    Npy c, r;
    if (pb_status s = c.open(dir + std::to_string(chunk) + ".codes.npy")) return s;
    if (pb_status s = r.open(dir + std::to_string(chunk) + ".residuals.npy")) return s;
    if (!c.is("i8") || c.count() != n_tokens)
        return pb_fail(PB_ERR_IO, "%lld.codes.npy must be <i8 [%lld]", chunk, n_tokens);
    if (!r.is("u1") || r.shape.size() != 2 || r.shape[0] != n_tokens || r.shape[1] != packed)
        return pb_fail(PB_ERR_IO, "%lld.residuals.npy must be u1 [%lld, %lld]", chunk, n_tokens, packed);
    codes.assign((const int64_t *)c.data, (const int64_t *)c.data + n_tokens);
    residuals.assign(r.data, r.data + (size_t)n_tokens * packed);
    return PB_OK;
}

pb_status pb_read_npy_f32(const std::string &path, long long &rows, long long &cols, std::vector<float> &out) {
    Npy a;
    if (pb_status s = a.open(path)) return s;
    if (!a.is("f4") || a.shape.size() != 2) return pb_fail(PB_ERR_IO, "%s must be <f4 [rows, cols]", path.c_str());
    rows = a.shape[0];
    cols = a.shape[1];
    out.assign((const float *)a.data, (const float *)a.data + a.count());
    return PB_OK;
}

namespace {

// A directory's inverted file: ivf.npy <i8 and ivf_lengths.npy, <i4 or (fast-plaid) <i8 narrowed into `store`
struct DirIvf {
    Npy ivf, ivfl;
    std::vector<int32_t> store;
    const int32_t *lengths = nullptr;
    pb_status open(const std::string &dir) {
        if (pb_status s = ivf.open(dir + "ivf.npy")) return s;
        if (pb_status s = ivfl.open(dir + "ivf_lengths.npy")) return s;
        if (!ivf.is("i8")) return pb_fail(PB_ERR_IO, "ivf.npy must be <i8");
        lengths = (const int32_t *)ivfl.data;
        if (ivfl.is("i8")) {
            const int64_t *src = (const int64_t *)ivfl.data;
            store.resize((size_t)ivfl.count());
            for (long long i = 0; i < ivfl.count(); ++i) {
                if (src[i] < 0 || src[i] > 0x7fffffffll) return pb_fail(PB_ERR_IO, "ivf_lengths.npy[%lld] out of range", i);
                store[(size_t)i] = (int32_t)src[i];
            }
            lengths = store.data();
        } else if (!ivfl.is("i4")) return pb_fail(PB_ERR_IO, "ivf_lengths.npy must be <i4 (next-plaid) or <i8 (fast-plaid)");
        return PB_OK;
    }
    pb_status check_sum(long long K) const {
        long long sum = 0;
        for (long long i = 0; i < K; ++i) sum += lengths[i];
        if (sum != ivf.count()) return pb_fail(PB_ERR_IO, "ivf.npy has %lld entries, ivf_lengths sum to %lld", ivf.count(), sum);
        return PB_OK;
    }
};

// The document layout of an index directory: metadata.json's num_chunks / nbits / num_embeddings (-1 when absent), and
// the doc lengths of every chunk (index.rs:1096-1104) with each chunk's token count.
struct DirLayout {
    double num_chunks = 0, nbits = 0, num_emb = -1;
    std::vector<int64_t> doclens;
    std::vector<long long> chunk_tokens;
    long long N = 0;

    pb_status read_metadata(const std::string &dir) {
        std::string meta;
        if (pb_status s = pb_read_text(dir + "metadata.json", meta)) return s;
        if (!pb_json_number(meta, "num_chunks", num_chunks) || !pb_json_number(meta, "nbits", nbits))
            return pb_fail(PB_ERR_IO, "metadata.json lacks num_chunks / nbits");
        pb_json_number(meta, "num_embeddings", num_emb);
        return PB_OK;
    }
    pb_status read_doclens(const std::string &dir) {
        for (int c = 0; c < (int)num_chunks; ++c) {
            const size_t first = doclens.size();
            if (pb_status s = pb_read_doclens(dir + "doclens." + std::to_string(c) + ".json", doclens)) return s;
            long long tok = 0;
            for (size_t i = first; i < doclens.size(); ++i) tok += doclens[i];
            chunk_tokens.push_back(tok);
        }
        for (long long t : chunk_tokens) N += t;
        if (num_emb >= 0 && (long long)num_emb != N)
            return pb_fail(PB_ERR_IO, "metadata.json num_embeddings=%lld but doclens sum to %lld", (long long)num_emb, N);
        return PB_OK;
    }
};

// pb_index_load of documents [doc_begin, doc_end) of the directory with pb_index_desc.flags; doc_end < 0 stands for every
// document
pb_status load_range(const char *index_dir, int32_t device, long long doc_begin, long long doc_end, int32_t flags,
                     pb_index **out) {
    const std::string dir = std::string(index_dir) + "/";
    DirLayout lay;
    if (pb_status s = lay.read_metadata(dir)) return s;
    const double num_chunks = lay.num_chunks, nbits = lay.nbits;

    Npy cent, wts;
    DirIvf div;
    if (pb_status s = cent.open(dir + "centroids.npy")) return s;
    if (pb_status s = wts.open(dir + "bucket_weights.npy")) return s;
    if (pb_status s = div.open(dir)) return s;
    const Npy &ivf = div.ivf, &ivfl = div.ivfl;
    const int32_t *ivfl_i32 = div.lengths;
    // fast-plaid directories (mmap.rs:1757-1811 converts them in place on the reference's first load): float tensors
    // as <f2, ivf_lengths as <i8, residuals described as <u1.  They are read as they are -- widened / narrowed in
    // memory, which gives the same values as the reference's conversion -- and never modified.
    std::vector<float> cent_store, wts_store;
    const float *cent_f32 = nullptr, *wts_f32 = nullptr;
    if (cent.shape.size() != 2) return pb_fail(PB_ERR_IO, "centroids.npy must be [K, dim]");
    if (pb_status s = as_f32(cent, "centroids.npy", cent_store, &cent_f32)) return s;
    if (pb_status s = as_f32(wts, "bucket_weights.npy", wts_store, &wts_f32)) return s;
    const long long K = cent.shape[0];
    const int dim = (int)cent.shape[1];
    const int nb = (int)nbits;
    if (nb <= 0 || 8 % nb != 0) return pb_fail(PB_ERR_INVALID, "nbits must be a divisor of 8, got %d", nb);
    if (wts.count() != (1ll << nb)) return pb_fail(PB_ERR_IO, "bucket_weights.npy has %lld entries, expected %d", wts.count(), 1 << nb);
    if (ivfl.count() != K) return pb_fail(PB_ERR_IO, "ivf_lengths.npy has %lld entries, centroids.npy %lld rows", ivfl.count(), K);

    if (pb_status s = lay.read_doclens(dir)) return s;
    const std::vector<int64_t> &doclens = lay.doclens;
    const std::vector<long long> &chunk_tokens = lay.chunk_tokens;
    const long long D = (long long)doclens.size();
    if (doc_end < 0) doc_end = D;
    if (doc_end > D)
        return pb_fail(PB_ERR_INVALID, "document range [%lld, %lld) outside the directory's %lld documents", doc_begin,
                       doc_end, D);
    // the range's tokens [t0, t1)
    long long t0 = 0, t1 = 0;
    for (long long i = 0; i < doc_end; ++i) (i < doc_begin ? t0 : t1) += doclens[i];
    t1 += t0;

    // the inverted file is not given to pb_index_open_begin: pb_index_upload_ivf_range slices ivf.npy on the device
    pb_index_desc d;
    memset(&d, 0, sizeof d);
    d.dim = dim;
    d.nbits = nb;
    d.num_centroids = K;
    d.num_documents = doc_end - doc_begin;
    d.num_embeddings = t1 - t0;
    d.centroids = cent_f32;
    d.bucket_weights = wts_f32;
    d.doc_lengths = doclens.data() + doc_begin;
    d.device = device;
    d.memory_space = PB_MEM_HOST;
    d.doc_id_base = doc_begin;
    d.flags = flags;
    if (pb_status s = div.check_sum(K)) return s;
    const long long packed = (long long)dim * nb / 8;
    // every chunk file is checked (header, dtype, shape, payload size) before the device is touched: a bad
    // directory fails here, not after tens of GB have been uploaded
    auto open_chunk = [&](int c, Npy &codes, Npy &res) -> pb_status {
        if (pb_status s = codes.open(dir + std::to_string(c) + ".codes.npy")) return s;
        if (pb_status s = res.open(dir + std::to_string(c) + ".residuals.npy")) return s;
        if (!codes.is("i8") || codes.count() != chunk_tokens[c])
            return pb_fail(PB_ERR_IO, "%d.codes.npy must be <i8 [%lld]", c, chunk_tokens[c]);
        if (!res.is("u1") || res.shape.size() != 2 || res.shape[0] != chunk_tokens[c] || res.shape[1] != packed)
            return pb_fail(PB_ERR_IO, "%d.residuals.npy must be u1 [%lld, %lld]", c, chunk_tokens[c], packed);
        return PB_OK;
    };
    for (int c = 0; c < (int)num_chunks; ++c) {
        if (chunk_tokens[c] == 0) continue;
        Npy codes, res;
        if (pb_status s = open_chunk(c, codes, res)) return s;
    }
    pb_index *ix = nullptr;
    if (pb_status s = pb_index_open_begin(&d, &ix)) return s;
    pb_status s = pb_index_upload_ivf_range(ix, (const int64_t *)ivf.data, ivfl_i32, ivf.count(), std::max(D, 1ll),
                                            doc_begin, doc_end);
    // the rows of each chunk that overlap [t0, t1), straight from the chunk's mapping
    for (long long c = 0, cs = 0; !s && c < (long long)num_chunks; cs += chunk_tokens[c++]) {
        const long long lo = std::max(cs, t0), hi = std::min(cs + chunk_tokens[c], t1);
        if (lo >= hi) continue;
        Npy codes, res;
        s = open_chunk((int)c, codes, res);
        if (!s)
            s = pb_index_upload_tokens(ix, lo - t0, (const int64_t *)codes.data + (lo - cs),
                                       res.data + (size_t)(lo - cs) * packed, hi - lo, PB_MEM_HOST);
    }
    if (!s) s = pb_index_finalize(ix);
    if (s) {
        pb_index_close(ix);
        return s;
    }
    *out = ix;
    return PB_OK;
}

}  // namespace

extern "C" pb_status pb_index_load(const char *index_dir, int32_t device, pb_index **out) {
    if (!index_dir || !out) return pb_fail(PB_ERR_INVALID, "null argument");
    *out = nullptr;
    return load_range(index_dir, device, 0, -1, 0, out);
}

extern "C" pb_status pb_index_load_range(const char *index_dir, int32_t device, int64_t doc_begin, int64_t doc_end,
                                         pb_index **out) {
    if (!index_dir || !out) return pb_fail(PB_ERR_INVALID, "null argument");
    *out = nullptr;
    if (doc_begin < 0 || doc_end < doc_begin)
        return pb_fail(PB_ERR_INVALID, "bad document range [%lld, %lld)", (long long)doc_begin, (long long)doc_end);
    return load_range(index_dir, device, doc_begin, doc_end, 0, out);
}

extern "C" pb_status pb_index_load_range_flags(const char *index_dir, int32_t device, int64_t doc_begin, int64_t doc_end,
                                               int32_t flags, pb_index **out) {
    if (!index_dir || !out) return pb_fail(PB_ERR_INVALID, "null argument");
    *out = nullptr;
    if (doc_begin < 0 || (doc_end >= 0 && doc_end < doc_begin))
        return pb_fail(PB_ERR_INVALID, "bad document range [%lld, %lld)", (long long)doc_begin, (long long)doc_end);
    return load_range(index_dir, device, doc_begin, doc_end, flags, out);
}

extern "C" pb_status pb_index_dir_shard_bounds(const char *index_dir, int32_t world, int64_t *out_bounds) {
    if (!index_dir || !out_bounds) return pb_fail(PB_ERR_INVALID, "null argument");
    if (world < 1) return pb_fail(PB_ERR_INVALID, "world must be at least 1, got %d", world);
    const std::string dir = std::string(index_dir) + "/";
    DirLayout lay;
    if (pb_status s = lay.read_metadata(dir)) return s;
    if (pb_status s = lay.read_doclens(dir)) return s;
    const long long D = (long long)lay.doclens.size();
    // bound r = min { d : doc_off[d] * world >= N * r }, in 128-bit so that no product overflows
    long long d = 0, off = 0;
    out_bounds[0] = 0;
    for (int r = 1; r < world; ++r) {
        while (d < D && (__int128)off * world < (__int128)lay.N * r) off += lay.doclens[d++];
        out_bounds[r] = d;
    }
    out_bounds[world] = D;
    return PB_OK;
}

pb_status pb_dir_patch_ivf(pb_index *ix, const char *index_dir, long long D, const uint32_t *bits, const long long *word_pre,
                           const uint64_t *keys, long long m, std::vector<int64_t> &ivf, std::vector<int32_t> &lengths) {
    DirIvf div;
    const long long K = pb_index_num_partitions(ix);
    if (pb_status s = div.open(std::string(index_dir) + "/")) return s;
    if (div.ivfl.count() != K) return pb_fail(PB_ERR_IO, "ivf_lengths.npy has %lld entries, the index %lld centroids", div.ivfl.count(), K);
    if (pb_status s = div.check_sum(K)) return s;
    return pb_index_patch_ivf(ix, (const int64_t *)div.ivf.data, div.lengths, div.ivf.count(), D, bits, word_pre, keys, m,
                              ivf, lengths);
}
