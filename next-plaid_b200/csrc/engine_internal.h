// engine_internal.h -- C++-side entry points shared between engine.cu, loader.cpp and builder.cpp (not exported).
#pragma once
#include "../../include/plaid_b200.h"

#include <string>
#include <vector>

pb_status pb_fail(pb_status s, const char *fmt, ...);
// pb_index_open without the per-token arrays; follow with pb_index_upload_tokens per chunk.
pb_status pb_index_open_begin(const pb_index_desc *d, pb_index **out);
pb_status pb_index_upload_tokens(pb_index *ix, long long tok_off, const int64_t *codes, const uint8_t *residuals,
                                 long long n, int space);
// call once after the last pb_index_upload_tokens
pb_status pb_index_finalize(pb_index *ix);
// For a handle begun without an inverted file: the part of a directory's inverted file (host ivf.npy <i8 [total],
// ivf_lengths [K], global ids, all checked against [0, limit)) that lies in docs [b, e), each list filtered in file
// order with ids minus b, instead of the one pb_index_finalize would build from the codes.
pb_status pb_index_upload_ivf_range(pb_index *ix, const int64_t *ivf, const int32_t *lengths, long long total,
                                    long long limit, long long b, long long e);
// The inverted file of a directory after a change, from its ivf.npy (host, as above, ids in [0, D)) to the host, i64
// global ids: with a deleted set (device bits / word_pre over the D docs) deleted ids leave the lists and survivors are
// renumbered (delete.rs:196-237); with the sorted (centroid << 32 | doc) device keys of m appended docs each list is
// followed by its new pairs as ids D + doc (update.rs:1000-1067).
pb_status pb_index_patch_ivf(pb_index *ix, const int64_t *file_ivf, const int32_t *file_lengths, long long total, long long D,
                             const uint32_t *bits, const long long *word_pre, const uint64_t *keys, long long m,
                             std::vector<int64_t> &ivf, std::vector<int32_t> &lengths);
// pb_index_patch_ivf on the directory's ivf.npy / ivf_lengths.npy as they are on disk
pb_status pb_dir_patch_ivf(pb_index *ix, const char *index_dir, long long D, const uint32_t *bits, const long long *word_pre,
                           const uint64_t *keys, long long m, std::vector<int64_t> &ivf, std::vector<int32_t> &lengths);

// The index directory, as the loader reads it: a whole file; a number of a flat JSON object; a doclens.{i}.json list;
// the chunk file pair {i}.codes.npy <i8 [n_tokens] / {i}.residuals.npy u1 [n_tokens][packed].
pb_status pb_read_text(const std::string &path, std::string &out);
bool pb_json_number(const std::string &j, const char *key, double &out);
pb_status pb_read_doclens(const std::string &path, std::vector<int64_t> &out);
pb_status pb_read_chunk(const std::string &dir, long long chunk, long long n_tokens, long long packed,
                        std::vector<int64_t> &codes, std::vector<uint8_t> &residuals);
// a 2-D <f4 NPY file (embeddings.npy, buffer.npy)
pb_status pb_read_npy_f32(const std::string &path, long long &rows, long long &cols, std::vector<float> &out);

// update_index's file changes (update.rs:794-1117, update_threshold = false) for n_docs documents appended to the
// index in index_dir, which holds old_D documents: chunk files in batches of batch_size docs (the first merged into a
// last chunk of < 2000 docs), the merged inverted file ivf / ivf_lengths (global ids), metadata.json, and removal of
// the merged_* caches.  codes i64 [sum doc_lengths], residuals packed [sum doc_lengths][dim*nbits/8].
pb_status pb_dir_append(const char *index_dir, long long old_D, long long K, int dim, int nbits, long long batch_size,
                        const int64_t *codes, const uint8_t *residuals, const int64_t *doc_lengths, long long n_docs,
                        const int64_t *ivf, long long ivf_total, const int32_t *ivf_lengths);

// PB_ERR_INVALID (PB_ERR_IO when unreadable) unless the directory's metadata.json holds D documents and nbits
pb_status pb_dir_check_documents(const char *index_dir, int nbits, long long D);

// delete_from_index's file changes (delete.rs:66-273) for the documents whose bit is set in `deleted` (one bit per doc
// of the old_D the directory holds): filtered chunk files and chunk metadata for every chunk with a deleted doc, the
// filtered inverted file ivf / ivf_lengths, metadata.json, removal of the merged_* caches, and the filtering of
// embeddings.npy / buffer.npy (clean_embeddings_files, delete.rs:286-398).
pb_status pb_dir_delete(const char *index_dir, long long old_D, long long K, int dim, int nbits, const uint32_t *deleted,
                        const int64_t *ivf, long long ivf_total, const int32_t *ivf_lengths);
