/*
 * oramacore_b200.h — C ABI of the H100-native (sm_90a) OramaCore search hot path.
 *
 * The reference (oramasearch/oramacore @ 666ab48) has no plugin / FFI boundary for this
 * path: the seam is Rust-to-Rust (SURVEY.md §8b).  Each entry point below names the
 * reference interface it replaces (file:line relative to the reference root).  Plain
 * pointers and sizes only; all `out_*` buffers are caller-allocated HOST memory; the
 * library owns every device allocation behind the opaque handles.  The shared library
 * (liboramacore_b200.so) is CUDA-only: there is no CPU fallback, every call fails with
 * OC_ERR_CUDA when no sm_90 device is usable.
 *
 * Status: 0 = OC_OK, <0 = error; text via oc_last_error() (thread-local, valid until the
 * next call on that thread).  Handles are Send+Sync: calls on one ctx are serialised
 * internally (one stream per ctx); different ctxs run concurrently.
 */
#ifndef ORAMACORE_B200_H
#define ORAMACORE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OC_OK 0
#define OC_ERR_INVALID (-1)     /* bad argument / shape                                   */
#define OC_ERR_CUDA (-2)        /* CUDA runtime failure (incl. "no device")               */
#define OC_ERR_OOM (-3)         /* device or host allocation failed                       */
#define OC_ERR_UNSUPPORTED (-4) /* e.g. limit+offset > OC_MAX_TOPK                        */
#define OC_ERR_COMM (-5)        /* NCCL failure / libnccl not loadable                    */

#define OC_MAX_TOPK 1024u       /* max limit+offset handled on device                     */
#define OC_MAX_TOKENS 32u       /* u32 token bitmask, token_score.rs:293                  */

#define OC_MODE_FULLTEXT 0      /* ScoreMode::FullText | Default, token_score.rs:472-484  */
#define OC_MODE_VECTOR 1        /* ScoreMode::Vector,             token_score.rs:485-494  */
#define OC_MODE_HYBRID 2        /* ScoreMode::Hybrid,             token_score.rs:495-503  */

#define OC_DTYPE_F32 0
#define OC_DTYPE_BF16 1         /* storage extension (reference stores f32, embedding_field.rs:232) */

typedef struct oc_ctx oc_ctx;   /* one device + stream + workspace (one per process/GPU)  */
typedef struct oc_emb oc_emb;   /* == one EmbeddingFieldStorage (embedding_field.rs:29-34) */
typedef struct oc_str oc_str;   /* == the StringFieldStorage set of one Index (string_field.rs:32-36) */
typedef struct oc_filter oc_filter; /* == a FilterResult<DocumentId> evaluated to a bitmap on the device (filter.rs:344-392) */
typedef struct oc_omc oc_omc;   /* == the OMC map of one Index (omc_committed + its log, index/mod.rs:604-627, 1720-1739) */

const char *oc_last_error(void);
int oc_version(void);
/* sizeof of {oc_search_params, oc_timing, oc_emb_info_t, oc_str_info_t} as compiled: lets a
 * binding (Rust repr(C), ctypes) verify its mirror of the structs at load time. */
void oc_abi_sizes(size_t out[4]);

/* ---- context ------------------------------------------------------------------------ */
/* Replaces nothing in the reference (it has no device); one ctx per GPU, one process per GPU. */
int oc_init(int device_id, oc_ctx **out);
void oc_shutdown(oc_ctx *ctx);
/* Number of SMs / device name, for bench reporting. */
int oc_device_info(oc_ctx *ctx, int *sm_count, size_t *hbm_bytes, char *name, size_t name_cap);

/* Document-sharded multi-GPU (SURVEY.md §8e; no reference analogue — the reference is
 * single-node).  Rank 0 creates the id, the host runtime broadcasts it, every rank joins.
 * After oc_comm_init, oc_search with params.sharded=1 all-gathers per-shard top-k over
 * NCCL/NVLink and merges on device; every rank receives the global answer.  When corpus df has
 * to be counted (a filter, multi-term tokens, tombstones: token_score.rs:262-275) the per-token
 * counters are summed across ranks with one ncclAllReduce before the idf is derived.  Every rank
 * must issue the same batch with the same flags: OC_SHARD_TOMBSTONES is set on ALL ranks while
 * ANY rank's string store holds uncommitted deletes (the host runtime routes deletes, so it knows). */
#define OC_SHARDED 1
#define OC_SHARD_TOMBSTONES 2
#define OC_SHARD_COUNT_DF 4      /* count corpus df across ranks (one ncclAllReduce) instead of using the per-term
                                    global_df tables: required, on EVERY rank, while any rank's string store lacks
                                    them (an oc_str_commit on a shard drops its table until oc_str_sync_global
                                    rebuilds it) */
#define OC_COMM_ID_BYTES 128
int oc_comm_unique_id(uint8_t out_id[OC_COMM_ID_BYTES]);
int oc_comm_init(oc_ctx *ctx, int world_size, int rank, const uint8_t id[OC_COMM_ID_BYTES]);
/* In-process group: ctxs[r] becomes rank r of `world` ranks (1..16 distinct contexts of this process, e.g. several
 * on one GPU, which NCCL refuses).  The collectives of a sharded oc_search then run on the calling threads through
 * host memory: each rank drains its own stream, copies its bytes to the host, waits for the other ranks (host
 * condition variable, fixed timeout) and copies the result back.  Every rank calls oc_search on its own thread.
 * Ranks that call different collectives (kind or size) all get OC_ERR_COMM and the group stays usable; a timeout,
 * or an oc_shutdown of one of the contexts, fails every later collective of the group. */
int oc_comm_init_local(oc_ctx *const *ctxs, int world);
/* Optional: direct NVLink exchange of the per-shard top-k records instead of the NCCL all-gather.  After
 * oc_comm_init every rank exports the CUDA-IPC handle of its receive window, the host runtime all-gathers the
 * blobs (world x OC_P2P_HANDLE_BYTES, rank order) and every rank imports them.  From then on the pack kernel of a
 * sharded oc_search stores each query's record straight into all ranks' windows (peer memory over NVLink /
 * NVSwitch) and bumps a per-query arrival counter; the merge kernel waits on the counters: no library collective
 * on the data path.  Batches whose records exceed the 1 MiB window fall back to ncclAllGather. */
#define OC_P2P_HANDLE_BYTES 128
int oc_comm_p2p_export(oc_ctx *ctx, uint8_t out_handle[OC_P2P_HANDLE_BYTES]);
int oc_comm_p2p_import(oc_ctx *ctx, const uint8_t *handles);

/* ---- embedding store ------------------------------------------------------------------
 * EmbeddingFieldStorage::new (embedding_field.rs:64-78): metric fixed = cosine;
 * rescale_e5 = Model::rescale_score for the E5 family (python/embeddings.rs:71-92).
 * An OC_DTYPE_F32 store also keeps an fp16 copy of its rows (each row scaled by a power of two), the operand of the
 * batched tensor-core sweep: 6 B per element in all instead of 4.  Scores are still exact fp32 arithmetic on the
 * stored rows.  OC_EMB_F16=0 in the environment at creation keeps no copy (the sweep then reads the fp32 rows through
 * tf32); if the copy cannot be allocated, the store drops it and is served the same way. */
int oc_emb_create(oc_ctx *ctx, uint32_t dim, int dtype, int rescale_e5, oc_emb **out);
void oc_emb_destroy(oc_emb *emb);
int oc_emb_reserve(oc_emb *emb, uint64_t n_rows);
/* EmbeddingFieldStorage::insert(DocumentId, Vec<Vec<f32>>) (embedding_field.rs:232-237),
 * batched: n vectors, doc_ids[i] may repeat (several chunks per document). rows = n x dim
 * row-major in the store's dtype, host memory. */
int oc_emb_insert(oc_emb *emb, const uint64_t *doc_ids, const void *rows, uint64_t n);
/* EmbeddingFieldStorage::delete (embedding_field.rs:240-242). */
int oc_emb_delete(oc_emb *emb, const uint64_t *doc_ids, uint64_t n);

typedef struct {
    uint64_t num_embeddings;  /* live vectors,   info().num_embeddings (embedding_field.rs:303-310) */
    uint64_t num_rows;        /* incl. tombstones */
    uint32_t dimensions;
    int dtype;
    uint64_t device_bytes;    /* rows, inverse norms, doc ids, and the fp16 copy with its row scales when kept */
} oc_emb_info_t;
int oc_emb_info(oc_emb *emb, oc_emb_info_t *out);

/* == EmbeddingFieldStorage compact() as Index::commit runs it (index/mod.rs:583-590): removes the rows oc_emb_delete
 * tombstoned, on the device and in place.  Live rows keep their relative order, so every search returns the ids,
 * score bits, counts and tie order it returned before; what changes is num_rows (== num_embeddings afterwards), the
 * bytes a sweep reads, and the room left for inserts.  The rows move through a staging window: the extra device
 * memory (workspace_bytes) is the window (32 MiB) plus a quarter byte per row of the store, each rounded up by a
 * quarter, never a second copy of the matrix; it is a ctx workspace, allocated for the call and freed at its end.  Rows below the first dead row are neither moved
 * nor read, and a store without dead rows launches nothing.
 * OC_EMB_COMPACT_SHRINK also gives the capacity beyond num_rows (rounded up to 64 rows) back by moving the store into
 * a smaller allocation; when that allocation cannot be made the store stays compacted at its old capacity and the
 * call still succeeds (device_bytes_after == device_bytes_before).  Without the flag the capacity is kept.
 * Runs under the ctx lock on the ctx stream and returns when the stream is idle; searches on the ctx serialise with
 * it.  A failure before the first row moves (OC_ERR_OOM for the workspace) leaves the store as it was.  There is no
 * rollback once rows move: the call then finishes or returns OC_ERR_CUDA, after which the store must be destroyed.
 * OC_ERR_INVALID: NULL store, unknown flag bits.  `out` may be NULL. */
#define OC_EMB_COMPACT_SHRINK 1u
typedef struct {
    uint64_t rows_before, rows_after;      /* num_rows before / after (after == num_embeddings)       */
    uint64_t rows_moved;                   /* live rows whose index changed                             */
    uint64_t device_bytes_before, device_bytes_after;   /* as oc_emb_info reports them                 */
    uint64_t workspace_bytes;              /* extra device memory the call held (0 when nothing ran)    */
    float device_ms;                       /* CUDA-event time of the device work, 0 when nothing ran    */
} oc_emb_compact_t;
int oc_emb_compact(oc_emb *emb, uint32_t flags, oc_emb_compact_t *out);

/* EmbeddingFieldStorage::search (embedding_field.rs:250-278) for B targets at once:
 * exact top-`limit` by cosine distance (== storage.search(target, limit, None) :255-266),
 * then similarity = 1 - distance, rescale, keep score >= similarity (:268-276).
 * filter_bits: NULL or a bitmap over DocumentId (FilterResult::contains, :54-61).
 * out_doc_ids/out_scores: B x limit, best first; out_counts[b] = hits kept (<= limit). */
int oc_emb_search(oc_emb *emb, const float *queries, uint32_t B, uint32_t limit, float similarity,
                  const uint64_t *filter_bits, uint64_t filter_nbits, uint64_t *out_doc_ids,
                  float *out_scores, uint32_t *out_counts);

/* ---- string (BM25F) store --------------------------------------------------------------
 * One oc_str holds all string fields of an Index over a shared row space
 * (row -> DocumentId).  Committed postings are handed over in CSR per field — what
 * StringFieldStorage::insert(DocumentId, IndexedValue{field_length:u16, terms}) accumulates
 * and compact() lays out (string_field.rs:155-177, 186-191). */
int oc_str_create(oc_ctx *ctx, uint32_t n_fields, oc_str **out);
void oc_str_destroy(oc_str *s);
/* row_doc_ids: NULL => DocumentId == row; must be ascending. document_count = N for idf
 * (Index::document_count, token_score.rs:221) — GLOBAL when sharded. */
int oc_str_set_rows(oc_str *s, uint64_t n_rows, const uint64_t *row_doc_ids, uint64_t document_count);
/* Postings of one field: term t owns [term_offsets[t], term_offsets[t+1]); rows ascending,
 * unique per term. avg_field_len = info().avg_field_length (string_field.rs:228-235),
 * global when sharded. global_df: NULL, or per-term corpus df across all shards (n_terms entries; a table read back
 * with oc_str_read_global_df may be longer than the field: pad term_offsets with its last entry to that size).
 * A shard loaded without tables gets them, and the corpus-wide averages, from oc_str_sync_global. */
int oc_str_load_field(oc_str *s, uint32_t field, float avg_field_len, uint32_t n_terms,
                      const uint64_t *term_offsets, const uint32_t *post_row, const uint16_t *post_tf,
                      const uint16_t *post_len, const uint32_t *global_df);
/* StringFieldStorage::insert(DocumentId, IndexedValue{field_length:u16, terms}) (string_field.rs:155-177),
 * with terms already resolved to the field's term ids by the host dictionary: buffered on the host,
 * visible to searches after oc_str_commit. Re-inserting a document (before or after a commit) replaces its
 * postings in that field: the last insert wins.  A term id may appear once per call. */
int oc_str_insert(oc_str *s, uint32_t field, uint64_t doc_id, uint16_t field_len, uint32_t n_terms,
                  const uint32_t *term_ids, const uint16_t *tfs);
/* == compact(version) (string_field.rs:186-191): merges pending inserts / deletes into the NEXT snapshot of the
 * device-resident layout (rows = ascending doc ids; avg_field_len and document_count refreshed unless the caller
 * owns the corpus-wide values, see oc_str_set_global; a shard's corpus-wide df tables are dropped: call
 * oc_str_sync_global on every rank afterwards) and publishes it with a pointer swap — the reference's
 * CURRENT + versions/<n> scheme (embedding_field.rs:91-95).  The build runs WITHOUT the context lock on the
 * store's own stream: oc_search keeps serving the previous version meanwhile.  A failed commit changes nothing
 * (the pending ops stay queued).  One commit at a time per store.  The merge runs on the device: its cost is
 * O(pending ops) on the host and one pass over the committed postings on the device, and the store keeps no host
 * copy of its postings.  Same as oc_str_commit_ex(s, NULL). */
int oc_str_commit(oc_str *s);
/* Statistics of one oc_str_commit_ex call. */
typedef struct {
    uint64_t rows_before, rows_after;          /* rows of the base and of the new snapshot                       */
    uint64_t postings_before, postings_after;  /* postings of all fields, base / new snapshot                    */
    uint64_t pending_postings;                 /* pending postings merged (after cancelled and replaced inserts) */
    uint64_t workspace_bytes;                  /* device memory the call held besides the new snapshot's arrays  */
    float device_ms;                           /* CUDA-event time of the device work on the store's load stream  */
    float wall_ms;                             /* the whole call, publishing included                             */
} oc_str_commit_t;
/* oc_str_commit, filling *out (may be NULL) when it succeeds.  OC_ERR_INVALID: a term id listed twice in one insert
 * of a document, or a commit already in flight; OC_ERR_OOM: no room for the new snapshot or the workspace.  Either
 * way nothing changes. */
int oc_str_commit_ex(oc_str *s, oc_str_commit_t *out);
/* Read-back of the published snapshot, the inverse of oc_str_set_rows + oc_str_load_field — what compact()
 * (string_field.rs:186-191) leaves on disk, so a caller can persist a committed version.  Each call reads one
 * snapshot; compare `version` across calls.  With NULL arrays they return the sizes; otherwise *n_rows (*n_terms,
 * *n_postings) is the capacity of the arrays on entry, and a capacity too small fails with OC_ERR_INVALID after
 * writing the sizes.  row_doc_ids gets the ascending doc id of every row (the identity when the store has no map);
 * term_offsets takes n_terms + 1 entries. */
int oc_str_read_rows(oc_str *s, uint64_t *n_rows, uint64_t *row_doc_ids, uint64_t *document_count, uint64_t *version);
int oc_str_read_field(oc_str *s, uint32_t field, float *avg_field_len, uint32_t *n_terms, uint64_t *n_postings,
                      uint64_t *term_offsets, uint32_t *post_row, uint16_t *post_tf, uint16_t *post_len);
/* StringFieldStorage::delete (string_field.rs:180-182).  Ops apply in call order like the reference's compact:
 * the committed rows of the document are tombstoned at once and its still-pending inserts are cancelled; an
 * insert after the delete is a new document. */
int oc_str_delete(oc_str *s, const uint64_t *doc_ids, uint64_t n);
/* The caller owns document_count (N of the idf = Index::document_count, token_score.rs:221 — it also counts
 * documents that have no string field, index/mod.rs:1460) and, when avg_field_len[n_fields] is given, the
 * corpus-wide average field lengths (this store is one shard of a larger index): oc_str_commit keeps the
 * caller's values instead of recomputing local ones (avg_field_len == NULL: averages stay locally computed).
 * Call again after commits to refresh them. */
int oc_str_set_global(oc_str *s, uint64_t document_count, const float *avg_field_len);
/* Rebuilds a shard's corpus-wide df tables and average field lengths from the stores of every rank of the ctx's comm
 * group (oc_comm_init / oc_comm_init_local): a collective.  Every rank calls it on its store after its own
 * oc_str_commit returned, at the same point of its sequence of sharded calls.  Under the ctx lock, on the ctx stream:
 *   1. the ranks all-gather {n_fields, rows, snapshot version}: different n_fields, or 2^32 rows or more in all (df
 *      is u32), give OC_ERR_INVALID on every rank;
 *   2. they all-gather each field's n_terms, and T_f = the largest;
 *   3. each rank writes the list lengths of its published snapshot (tombstoned rows included), zero-padded to T_f,
 *      and per field the sum and count of its non-zero row lengths (one length per row, read from the postings on
 *      the device, exact in u64), all-gathers those sums with its allocation / kernel status (a bad one on any rank
 *      is every rank's return code, OC_ERR_OOM or OC_ERR_CUDA), and all-reduces the df buffer (sum T_f counters);
 *   4. installs on the snapshot read in 3: each field's df table (T_f entries: a term this shard has no posting of
 *      counts as an empty list, so every rank takes the same df decisions), avg_field_len = the sums' quotient as
 *      oc_str_commit computes it (a field without a non-zero length keeps its value), a new snapshot identity.
 * A rank whose ctx has no comm gets OC_ERR_COMM; a refused call changes nothing and leaves the group usable.
 * N (document_count) stays the caller's: it also counts documents with no string field.  A later oc_str_commit
 * drops the tables again (OC_SHARD_COUNT_DF keeps its meaning) and handles the averages as before; a commit in
 * flight during the sync publishes after it the same way.  oc_str_set_global(N, NULL) keeps tables and averages.
 * out (may be NULL): */
typedef struct {
    uint64_t version;          /* the snapshot the values were installed on                                  */
    uint64_t rows_global;      /* sum of the ranks' rows                                                     */
    uint64_t bytes_reduced;    /* this rank's contribution: df table entries x 4 + the length pairs (16 B each) */
    float device_ms;           /* CUDA-event time of the length sums and of the df all-reduce with its read-back */
    float wall_ms;             /* the whole call                                                              */
} oc_str_sync_t;
int oc_str_sync_global(oc_str *s, oc_str_sync_t *out);
/* Host read-back of one field's installed df table: df NULL -> *n_terms = its size (0: no table); otherwise *n_terms
 * is df's capacity on entry (too small: OC_ERR_INVALID after writing the size).  The array oc_str_load_field's
 * global_df takes, so a persisted shard reloads with it. */
int oc_str_read_global_df(oc_str *s, uint32_t field, uint32_t *n_terms, uint32_t *df);

typedef struct {
    uint64_t total_documents;  /* rows                              */
    uint64_t total_postings;
    uint64_t unique_terms_count;
    uint32_t n_fields;
    uint64_t device_bytes;
    uint64_t version;          /* published snapshot, bumped by every load / commit (== CURRENT)  */
    uint64_t pending_postings; /* inserted, not yet committed (cf. pending_ops, embedding_field.rs:303-310) */
} oc_str_info_t;
int oc_str_info(oc_str *s, oc_str_info_t *out);

/* ---- search() ---------------------------------------------------------------------------
 * TokenScoreContext::execute (token_score.rs:460-509) + apply_omc_multipliers
 * (search.rs:39-48) + count (search.rs:482) + sort_token_scores/top_n (sort.rs:17-46,
 * 260-279) + skip(offset).take(limit) (search.rs:494-498), for a batch of B queries.
 *
 * Query text is resolved to index terms on the host (tokenise+stem token_score.rs:196-209;
 * prefix/Levenshtein expansion inside StringStorage); the ABI takes, per query, its tokens,
 * and per token the expanded (field, term id, weight) list, weight = field boost x
 * exact-match factor (the "ntf already includes boost" contract, token_score.rs:180-185). */
typedef struct {
    int mode;                          /* OC_MODE_*                                         */
    uint32_t n_queries;                /* B                                                  */
    uint32_t limit, offset;            /* Limit / SearchOffset (types.rs:747-756)            */
    float similarity;                  /* Similarity (types.rs:878-901); vector & hybrid     */
    float threshold;                   /* Threshold (types.rs:859-876); < 0 => None          */
    float bm25_k, bm25_b;              /* 1.2 / 0.75 (token_score.rs:283; bm25.rs:56-63)     */
    const float *q_vecs;               /* B x dim fp32 (vector, hybrid) or NULL              */
    const uint32_t *q_token_offsets;   /* B+1 (fulltext, hybrid) or NULL                     */
    const uint32_t *token_term_offsets;/* n_tokens+1                                         */
    const uint32_t *term_field;        /* per expanded term                                  */
    const uint32_t *term_id;
    const float *term_weight;
    const uint64_t *filter_bits;       /* NULL or bitmap over DocumentId                     */
    uint64_t filter_nbits;
    const uint64_t *omc_doc_ids;       /* OMC multipliers sorted by doc id (index/mod.rs:1720-1739) */
    const float *omc_mult;
    uint64_t n_omc;
    int sharded;                       /* OC_SHARDED [| OC_SHARD_TOMBSTONES | OC_SHARD_COUNT_DF] => merge across oc_comm ranks */
    uint32_t vector_limit;             /* 0 => limit.  Candidate depth of the vector stage = limit_hint, which the
                                          reference keeps at `limit` while top_n takes limit+offset (search.rs:330-336):
                                          a caller that needs the rows [0, limit+offset) of one index (multi-index
                                          union, oc_merge_results) asks for limit' = limit+offset, vector_limit = limit */
    const struct oc_filter *filter;    /* NULL, or a device-resident DocumentId bitmap (oc_filter_*): takes precedence
                                          over filter_bits and is not re-uploaded per call                           */
    const struct oc_filter *const *q_filters;  /* NULL, or B entries: query b is filtered by q_filters[b] (NULL = none) */
    const struct oc_query_params *q_params;    /* NULL, or B entries: query b's own mode, limit, offset, similarity,
                                                  threshold and vector_limit (see below)                          */
    const struct oc_where *q_where;            /* NULL, or query b's where-clause as a program, evaluated inside the
                                                  call (see "where programs" below); same meaning as q_filters     */
    const struct oc_omc *omc;                  /* NULL, or the index's OMC store (oc_omc_*): the call is byte for byte
                                                  the call with omc_doc_ids / omc_mult / n_omc set to the store's
                                                  published version, without a per-call upload; not together with
                                                  n_omc != 0 (see "OMC store" below)                               */
} oc_search_params;

/* One query's scalar parameters (SearchParams, types.rs:1381-1409, with FulltextMode / VectorMode / HybridMode,
 * types.rs:837-912): the fields of oc_search_params with the same names, for one query. */
typedef struct oc_query_params {
    int mode;              /* OC_MODE_*                                      */
    uint32_t limit, offset;
    float similarity;      /* vector / hybrid                                */
    float threshold;       /* < 0 => None                                    */
    uint32_t vector_limit; /* 0 => limit (as oc_search_params.vector_limit)  */
} oc_query_params;

/* out_doc_ids/out_scores: B x limit (best first, after offset); out_n[b] hits written;
 * out_count[b] = all matching documents. emb may be NULL for fulltext, str NULL for vector.
 *
 * Per-query where-filters (q_filters): every request of the reference carries its own where-filter
 * (SearchParams.where_filter), evaluated per request and passed into that request's scoring.  With q_filters set,
 * query b is scored exactly as if it were alone in an oc_search with p->filter = q_filters[b]: the vector stage,
 * the fulltext stage with the corpus df counted under that query's filter (token_score.rs:262-275), hybrid fusion,
 * OMC, count and offset / limit.  The result is byte-identical: same ids, same score bits, same count.
 *   - Entries may repeat; the library deduplicates by handle and builds one row bitmap per distinct handle over each
 *     store's rows (K distinct handles: K x rows / 8 bytes per store).  Each entry has its own nbits (ids >= nbits
 *     do not pass).  All entries NULL: an unfiltered search; every entry the same handle: the p->filter path.
 *   - OC_ERR_INVALID: q_filters together with filter or filter_bits, a handle of another ctx.
 *     OC_ERR_UNSUPPORTED: sharded.  A refused call creates nothing and writes no output.
 *   - oc_search_q_sorted takes q_filters together with a sort and pins per query, oc_search_q_groups together with
 *     groups, a sort and pins per query;
 *   - oc_search_groups*, oc_search_pinned and oc_search_sorted refuse q_filters with OC_ERR_UNSUPPORTED;
 *     oc_search_facets ignores it as it ignores filter (facets are scored without the where-filter).
 *
 * Per-query parameters (q_params): every request of the reference sets its own mode, limit, offset, similarity and
 * threshold.  With q_params set, query b's outputs — ids, score bits, n, count, and in the calls below its sort values,
 * pin scores / present flags, group rows and facet counts — are byte for byte what it gets alone: B = 1 with
 * p->mode / limit / offset / similarity / threshold / vector_limit taken from q_params[b], together with its own
 * filter, sort, items, groups and facets.  So a batch whose entries all equal p's scalars gives the plain call's
 * outputs.  Taken by oc_search, oc_search_q_sorted, oc_search_q_groups and oc_search_q_facets.
 *   - Layout: p->limit is the row stride of the hit arrays (out_doc_ids, out_scores, out_sort_values) and must be at
 *     least every entry's limit; entries past out_n[b] are 0.  p->mode, offset, similarity, threshold and
 *     vector_limit are ignored; bm25_k, bm25_b, OMC, filter / filter_bits / q_filters and sharded stay batch-wide.
 *   - Inputs: emb and q_vecs are needed when some entry has a vector part (q_vecs keeps B rows; the rows of fulltext
 *     entries are not read), str and q_token_offsets when some entry has a text part (the token ranges of vector
 *     entries are ignored).
 *   - Refusals (nothing written): every check a query's scalars get alone applies to its entry (unknown mode, limit 0
 *     where the entry point refuses it, the limit + offset, 2 x (limit + offset) and vector_limit bounds, a missing
 *     store or array for its mode); OC_ERR_INVALID: an entry's limit above p->limit; OC_ERR_UNSUPPORTED: p->sharded,
 *     and q_params given to oc_search_pinned, oc_search_sorted, oc_search_groups* or oc_search_facets.
 *   - Cost: one sweep of the embedding store serves the entries with a vector part, at their largest depth; the
 *     fulltext stage keeps every query's candidates at the largest limit + offset.  One entry with a threshold routes
 *     the batch's fulltext stage to the threshold scorer, one vector depth above 128 the vector sweep to the exact
 *     path. */
int oc_search(oc_ctx *ctx, oc_emb *emb, oc_str *str, const oc_search_params *p,
              uint64_t *out_doc_ids, float *out_scores, uint32_t *out_n, uint64_t *out_count);

/* ---- filters on the device -------------------------------------------------------------------------
 * FilterContext::execute_filter (read/index/filter.rs:344-392) yields a FilterResult tree: And / Or / Not over
 * plain DocumentId sets (:351-362, 378-389), consulted by the scorers through contains(doc)
 * (embedding_field.rs:54-61, string_field.rs:66-69).  Here a FilterResult is a bitmap over DocumentId
 * [0, nbits) that lives on the device: build the leaves from id lists, combine with And / Or / Not (word-wise
 * kernels), hand the handle to any number of oc_search / oc_search_facets calls (no per-call upload).
 * execute_filter's own rule — AND the where-filter with NOT(uncommitted deletes) — is oc_filter_and +
 * oc_filter_not over an id leaf of the deleted documents.
 * oc_filter_and(a, b) is oc_filter_from_where (below) of the program {FILTER a, FILTER b, AND 2} over a's nbits,
 * oc_filter_or the same with OR 2, and oc_filter_not(a) that of {FILTER a, NOT}: a handle of another ctx, or b of
 * another nbits than a, is refused with OC_ERR_INVALID and nothing is created. */
int oc_filter_from_ids(oc_ctx *ctx, const uint64_t *doc_ids, uint64_t n, uint64_t nbits, oc_filter **out);  /* PlainFilterResult::from_iter; ids >= nbits ignored */
int oc_filter_from_bits(oc_ctx *ctx, const uint64_t *bits, uint64_t nbits, oc_filter **out);
int oc_filter_and(const oc_filter *a, const oc_filter *b, oc_filter **out);   /* FilterResult::And */
int oc_filter_or(const oc_filter *a, const oc_filter *b, oc_filter **out);    /* FilterResult::Or  */
int oc_filter_not(const oc_filter *a, oc_filter **out);                       /* FilterResult::Not (within [0, nbits)) */
int oc_filter_count(const oc_filter *f, uint64_t *out);                       /* documents that pass */
/* The DocumentId space [0, nbits) of a handle: a leaf of a facet store or geopoint field takes the nbits of the version
 * it was built on, which a concurrent commit may grow. */
int oc_filter_nbits(const oc_filter *f, uint64_t *out);
int oc_filter_read(const oc_filter *f, uint64_t *out_bits /* (nbits+63)/64 words */);
void oc_filter_destroy(oc_filter *f);

/* ---- geopoint where-filter leaves -----------------------------------------------------------------
 * GeoPointFieldStorage::filter (read/index/geopoint_field.rs:179-229) for Filter::GeoPoint (read/index/filter.rs:125-139):
 * the documents of a geopoint field with a point inside (or outside) a radius or a polygon, as an ordinary oc_filter
 * over [0, nbits) of the field's ctx that combines with oc_filter_and / or / not and goes to any search as p->filter.
 * Each call is oc_filter_from_where (below) of a program of one OC_WHERE_GEO_RADIUS / OC_WHERE_GEO_POLYGON node over the
 * field's nbits: one scan of the field's points on the device.
 *   - Coordinates: degrees, latitude in [-90, 90], longitude in [-180, 180], both finite (FieldsGeoPoint::new refuses
 *     anything else).  The reference widens its f32 API values to f64; the caller does the same before calling here.
 *   - A field holds (document, point) entries; a document may have several points (GeoPointIndexedValue::Array).  A
 *     document is in a leaf when AT LEAST ONE of its points satisfies the leaf's predicate, also for inside = 0, whose
 *     predicate is "outside" (assumption).  A document with no point is in neither leaf.  Ids >= nbits are ignored.
 * The geometry lives in the un-vendored oramacore_fields crate; this library assumes:
 *   - radius: great-circle distance on a sphere of radius OC_GEO_EARTH_RADIUS_M; inside when d <= radius (boundary
 *     included), outside when d > radius; radius >= pi x R puts every point inside.  Evaluated as the chord test
 *     |u_p - u_c|^2 <= 4 sin^2(radius / 2R) on unit vectors, so points within ~1e-9 relative of the boundary may fall
 *     on either side.  radius_m is value.to_meter(unit) computed in f32 and widened (types.rs:2159-2170).
 *   - polygon: the even-odd ray-crossing test (PNPOLY) in planar (lon, lat) degrees over the edges (v[i-1], v[i]),
 *     cyclic (closed implicitly; a repeated closing vertex is harmless), evaluated in f64 as
 *     (yi > y) != (yj > y) && x < (xj - xi) * (y - yi) / (yj - yi) + xi, in that order, without FMA contraction.  Edges
 *     are not geodesic and do not wrap at +-180.  "Outside" is the negation of the test for each point.
 * OC_ERR_INVALID, creating nothing: invalid coordinates in the field or the query, a radius that is NaN, infinite or
 * negative, fewer than 3 or more than OC_GEO_MAX_VERTICES vertices (the kernel stages them in shared memory). */
#define OC_GEO_EARTH_RADIUS_M 6371000.0
#define OC_GEO_MAX_VERTICES 2048u
/* Statistics of one oc_facets_commit_ex / oc_geo_field_commit_ex call. */
typedef struct {
    uint64_t version;                          /* version this call published (1 = the first commit)       */
    uint64_t rows_kept, rows_dropped, rows_added;   /* entries of all fields: committed kept / removed, inserted */
    uint64_t workspace_bytes;                  /* largest device workspace of one field                      */
    float device_ms;                           /* CUDA-event time of the merge kernels, scans and their copies */
    float wall_ms;                             /* the whole call, publishing included                        */
} oc_filter_commit_t;
typedef struct oc_geo_field oc_geo_field;
/* n entries (doc_ids[i], lat[i], lon[i]); n = 0 gives empty leaves.  Sorted by document id and kept on the device as
 * 48 B per point (unit vector, lat / lon, id).  A changed field is committed with oc_geo_field_commit_ex
 * below. */
int oc_geo_field_create(oc_ctx *ctx, uint64_t nbits, uint64_t n, const uint64_t *doc_ids, const double *lat,
                        const double *lon, oc_geo_field **out);
void oc_geo_field_destroy(oc_geo_field *g);
/* compact() of a geopoint field: oc_geo_field_insert queues points (checked as oc_geo_field_create checks them, before
 * anything is queued), oc_geo_field_delete removes every point of the documents, in call order as for oc_facets_*, and
 * oc_geo_field_commit_ex merges them into the next version on the device with the contract, cost and refusals of
 * oc_facets_commit_ex (48 B per point; workspace 24 B per committed point, about 64 B per queued one).  A document's
 * points keep their order: committed first, then queued ones in call order.  The unit vectors of the queued points are
 * computed on the host as oc_geo_field_create computes them, so both give the same bits.  oc_geo_field_read reads the
 * published points back in their order (NULL arrays: the size; otherwise *n is the capacity on entry). */
int oc_geo_field_insert(oc_geo_field *g, uint64_t n, const uint64_t *doc_ids, const double *lat, const double *lon);
int oc_geo_field_delete(oc_geo_field *g, uint64_t n, const uint64_t *doc_ids);
int oc_geo_field_commit_ex(oc_geo_field *g, uint64_t new_nbits, oc_filter_commit_t *out);
int oc_geo_field_read(oc_geo_field *g, uint64_t *n, uint64_t *doc_ids, double *lat, double *lon);
/* GeoFilterOp::Radius / OutsideRadius: inside != 0 => points with d <= radius_m, else points with d > radius_m. */
int oc_filter_geo_radius(const oc_geo_field *g, double lat, double lon, double radius_m, int inside, oc_filter **out);
/* GeoFilterOp::Polygon / OutsidePolygon over the vertices (lat[k], lon[k]), k < n_vertices. */
int oc_filter_geo_polygon(const oc_geo_field *g, const double *lat, const double *lon, uint32_t n_vertices, int inside,
                          oc_filter **out);

/* ---- facets over the score set ------------------------------------------------------------------
 * FacetContext::execute (read/index/facet.rs:147-209): for each requested variant of a filter field — bool
 * true / false (bool_field.rs:182-208), a number range [from, to], both ends inclusive (number_field.rs:368-387,
 * NumberFilter::Between), a string_filter key (string_filter_field.rs:175-193) — the number of the variant's
 * documents that are keys of the score map.  The store keeps, per field, the variants' document lists on the
 * device (number fields: documents sorted by value, so a range is a slice); a search in facet mode makes the tile
 * scorer emit the bitmap of matched documents (+ the vector hits) and one kernel counts every (query, variant): each
 * distinct document slice is read once, against every query that asks for it.
 * As in the reference (search.rs:361-396) the score map is computed WITHOUT the where-filter (uncommitted deletes
 * stay excluded), so p->filter_bits / p->filter are ignored here: hits come from oc_search, facets from this call.
 * A document may be listed under several variants (array values).  nbits: DocumentId space [0, nbits). */
typedef struct oc_facets oc_facets;
typedef struct {
    uint32_t field;     /* id returned by oc_facets_add_*                                     */
    uint32_t variant;   /* bool / string fields: variant index                                */
    double from, to;    /* number fields: inclusive range                                     */
} oc_facet_req;
int oc_facets_create(oc_ctx *ctx, uint64_t nbits, oc_facets **out);
void oc_facets_destroy(oc_facets *f);
int oc_facets_add_field(oc_facets *f, uint32_t n_variants, const uint64_t *variant_offsets /* n+1 */, const uint64_t *doc_ids,
                        uint32_t *out_field);
/* The store keeps each variant's documents ascending, and a number field's entries ascending by value (-0.0 before
 * +0.0) then by document: input in another order inside a variant or a run of equal values is sorted on the host. */
int oc_facets_add_number_field(oc_facets *f, uint64_t n, const double *values_sorted, const uint64_t *doc_ids, uint32_t *out_field);

/* ---- filter-field commit -------------------------------------------------------------------------
 * compact() of the bool, string_filter, number and date fields (read/index/mod.rs:537-580) without a host rebuild:
 * pending ops queue on the host, in call order, and oc_facets_commit_ex merges them into the next version of every
 * field's device arrays.  Ops are not visible to searches before the commit.
 *   - oc_facets_insert_variants: (doc_ids[i], variants[i]) entries of a bool or string_filter field.  OC_FACET_UNIQUE
 *     gives set semantics: the entry is skipped when the field already holds it (committed and not removed, or queued
 *     earlier), as for a bool field.  Without it a document may hold a variant several times (array values).
 *   - oc_facets_add_variant: a new string_filter key; it gets the next variant index.  Variant indices never move, so
 *     oc_facet_req.variant and where-program nodes stay meaningful across commits.  The variant is empty until a
 *     commit publishes entries for it.
 *   - oc_facets_insert_numbers: (doc_ids[i], values[i]) entries of a number or date field; NaN is refused.
 *   - oc_facets_clear: removes every value of the documents in one field (a replaced value, FilterBool).
 *   - oc_facets_delete: removes every value of the documents in every field.
 * A removal applies to the committed entries and to the queued inserts before it, not to later inserts: a delete
 * followed by an insert of the same document keeps the insert.
 * oc_facets_commit_ex builds the next version from the previous version's DEVICE arrays on the handle's own stream,
 * outside the ctx lock: searches, leaves, where programs and oc_group_by_create keep running on the previous version
 * meanwhile, and the next one is published under the ctx lock once the ctx stream has drained.  new_nbits >= nbits
 * may grow the DocumentId space; every queued document must be below it.  Order inside a field after a commit:
 * variant-major with ascending documents (CSR), or ascending value, -0.0 before +0.0, then ascending document (number
 * and date fields).  A store built by oc_facets_add_* may order equal values differently; every consumer reads a
 * slice as a set.  The host copy of a number field's values is replaced by a copy of the merge result.
 * Cost: host O(pending log pending), plus a device-to-host copy of each changed number field's values; device one
 * pass over each changed field (a field with no queued insert and no removal is left as it is).  Workspace per
 * changed field, freed before the call returns: 24 B per committed entry, about 40 B per queued insert, 8 B per
 * removed document and the CUB scan storage.  Limit: fewer than 2^31 - 1 committed + queued entries per field.
 * OC_ERR_INVALID, changing nothing and keeping every op queued: new_nbits < nbits, a queued document >= new_nbits, a
 * commit of the handle already in flight; OC_ERR_OOM: no room for the workspace or the next version.  One commit at a
 * time per handle; oc_facets_add_* is refused while one is in flight. */
#define OC_FACET_UNIQUE 1u
int oc_facets_insert_variants(oc_facets *f, uint32_t field, uint64_t n, const uint64_t *doc_ids, const uint32_t *variants, uint32_t flags);
int oc_facets_add_variant(oc_facets *f, uint32_t field, uint32_t *variant_out);
int oc_facets_insert_numbers(oc_facets *f, uint32_t field, uint64_t n, const uint64_t *doc_ids, const double *values);
int oc_facets_clear(oc_facets *f, uint32_t field, uint64_t n, const uint64_t *doc_ids);
int oc_facets_delete(oc_facets *f, uint64_t n, const uint64_t *doc_ids);
int oc_facets_commit_ex(oc_facets *f, uint64_t new_nbits, oc_filter_commit_t *out);
/* Read-back of one field of the published version, as oc_facets_add_field / oc_facets_add_number_field take it.  With
 * every array NULL it returns the sizes (*n_variants = 0 for a number field).  Otherwise it fills the arrays given, and
 * *n_entries (doc_ids, values) and *n_variants (offsets) are their capacities on entry; offsets takes n_variants + 1
 * entries (the host copy: no device read), values (number fields) n_entries. */
int oc_facets_read_field(oc_facets *f, uint32_t field, uint32_t *n_variants, uint64_t *n_entries, uint64_t *offsets, double *values,
                         uint64_t *doc_ids);

/* ---- OMC store --------------------------------------------------------------------------------------
 * The OMC ("Orama Custom Multiplier") map of one index (omc_committed, read/index/mod.rs:604-627, 1720-1739): a score
 * multiplier per document, applied to every score map before count and top-N (read/search.rs:39-48, 340-343).  One
 * handle per index, on one ctx.  The published version lives on the device as doc[n] (strictly ascending) and
 * mult[n]; a search with oc_search_params.omc = the handle reads it there.
 *   - oc_omc_set queues (doc_ids[i], mults[i]) entries, oc_omc_delete queues removals.  Both apply in call order at the
 *     next commit; the last op for a document wins.  Values: any finite f32 (as the array path takes them); NaN and
 *     +-inf are refused with OC_ERR_INVALID and nothing of the call is queued.  The store does not drop zero or
 *     negative values: the reference's write side does that before it emits Index2 (write/index/mod.rs:451-458).
 *   - oc_omc_commit_ex merges the queue into the next version on the device, with no host copy of the map: the ops
 *     are radix-sorted by (document, call order), the last op per document is kept, and one pass merges them with the
 *     previous version.  The merge runs on the handle's own stream outside the ctx lock; the next version is published
 *     under the ctx lock once the ctx stream has drained, so a search holds one whole version, old or new.  A commit
 *     with no queued op publishes the same entries under the next version number.  Statistics in oc_filter_commit_t:
 *     rows_kept (committed entries kept as they were), rows_dropped (committed entries deleted or replaced), rows_added
 *     (entries written from the queue).  Workspace, freed before the call returns: about 30 B per queued op plus 8 B
 *     per committed entry and the CUB sort and scan storage.  Limit: fewer than 2^31 - 1 committed + queued entries.
 *     OC_ERR_INVALID, changing nothing and keeping every op queued: a commit of the handle already in flight;
 *     OC_ERR_OOM: no room for the workspace or the next version.
 *   - oc_omc_read reads the published version back.  With doc_ids and mults NULL it returns the size in *n; otherwise
 *     *n is their capacity on entry (too small: OC_ERR_INVALID after writing the size).  version (may be NULL): 0
 *     before the first commit, then the number the last commit published.
 * Searches: every search entry point (oc_search, oc_search_facets, oc_search_groups*, oc_search_pinned,
 * oc_search_sorted, the q_* calls and the sharded search) takes p->omc.  The ids, score bits, n, count, sort values, pin
 * outputs, group rows and facet counts are byte for byte those of the same call with omc_doc_ids / omc_mult / n_omc set
 * to the version oc_omc_read returns.  The tile scorers read the version's documents as string rows: the first search
 * after a commit of the handle or an oc_str_commit of its string store builds that list on the device and keeps it on
 * the handle (one device-to-host copy of its length, the only synchronisation this adds); other searches do no host
 * work and no upload for OMC.  OC_ERR_INVALID, nothing written: p->omc together with n_omc != 0, a handle of another
 * ctx.  Sharded searches: the shard merge applies the multipliers to every rank's candidates, so each rank's handle
 * must hold the whole index's map (a caller contract, as for the replicated df tables; not verified).
 * oc_omc_destroy: no search or commit of the handle may be in flight. */
int oc_omc_create(oc_ctx *ctx, oc_omc **out);
void oc_omc_destroy(oc_omc *omc);
int oc_omc_set(oc_omc *omc, const uint64_t *doc_ids, const float *mults, uint64_t n);
int oc_omc_delete(oc_omc *omc, const uint64_t *doc_ids, uint64_t n);
int oc_omc_commit_ex(oc_omc *omc, oc_filter_commit_t *out);
int oc_omc_read(oc_omc *omc, uint64_t *n, uint64_t *doc_ids, float *mults, uint64_t *version);

/* where-filter leaves over a filter field of a facet store (read/index/filter.rs:49-124); the leaf's nbits is the store's.
 * An ordinary oc_filter over the facets' ctx, for oc_filter_and / or / not and any search.  A document is in a leaf
 * when AT LEAST ONE of its values passes.  Each call is oc_filter_from_where (below) of a program of one
 * OC_WHERE_VARIANT / OC_WHERE_RANGE node over the store's nbits: the slice of the field is found by a binary search of
 * the host copy of its values, then the device slice is scattered into a zeroed bitmap.  Ids >= nbits are ignored.
 *   - oc_filter_facet_variant: the documents of variant `variant` of a bool or string_filter field (bool_field.rs:163-166,
 *     string_filter_field.rs:165-167).  Bool variants are 0 = true, 1 = false; a string_filter variant is one key.
 *   - oc_filter_facet_range: the documents of a number field with a value v in the interval [lo, hi], compared as
 *     f64 (IEEE: -0.0 == 0.0); OC_RANGE_LO_OPEN / OC_RANGE_HI_OPEN make that end open.  lo > hi is empty; +-inf are
 *     allowed.  NumberFilter and DateFilter map onto it (number_field.rs:555-642, date_field.rs:271-280):
 *     eq b = [b, b], gt b = (b, +inf], gte b = [b, +inf], lt b = [-inf, b), lte b = [-inf, b], between (a, b) = [a, b],
 *     with the bound widened to f64 (a Number is I32 or F32; a date is its millisecond timestamp).  The reference keeps
 *     integer and float values apart and converts F32 bounds for the integer values with ceil / floor and an EPSILON
 *     test; for integer values |v| <= 2^53 that selects what this interval selects, except that a nonzero F32 bound
 *     with |b| < 2^-52 counts as 0 there, so eq and lt / gt by such a bound differ from this interval at v = 0
 *     (deliberate: the interval is the plain comparison with the given bound).
 * OC_ERR_INVALID, creating nothing (*out untouched): NULL arguments, a field or variant out of range, a variant leaf on
 * a number field or a range leaf on a bool / string_filter field, a NaN bound, unknown flag bits. */
int oc_filter_facet_variant(const oc_facets *f, uint32_t field, uint32_t variant, oc_filter **out);
#define OC_RANGE_LO_OPEN 1u
#define OC_RANGE_HI_OPEN 2u
int oc_filter_facet_range(const oc_facets *f, uint32_t field, double lo, double hi, uint32_t flags, oc_filter **out);

/* ---- where programs ------------------------------------------------------------------------------
 * A where-clause as a postfix program, evaluated inside a search call (oc_search_params.q_where) or into a handle
 * (oc_filter_from_where, which every leaf call above and oc_filter_and / or / not use).  Query b's program is
 * nodes[q_node_offsets[b] .. q_node_offsets[b + 1]); an empty range leaves the query unfiltered.  Each node pushes one
 * bitmap over [0, nbits) or combines the top of the stack:
 *   OC_WHERE_NONE         the empty set
 *   OC_WHERE_VARIANT      src = oc_facets *: the documents of variant arg of the store's bool / string_filter field
 *   OC_WHERE_RANGE        src = oc_facets *: the documents of the store's number field with a value in [a, b], an end
 *                         open under the OC_RANGE_* flags in arg (the rules of oc_filter_facet_range above)
 *   OC_WHERE_GEO_RADIUS   src = oc_geo_field *: the documents with a point within c = radius_m metres of (a = lat,
 *                         b = lon), or with arg = inside = 0 a point beyond it (geometry: "geopoint where-filter leaves")
 *   OC_WHERE_GEO_POLYGON  src = oc_geo_field *: the documents with a point inside the polygon of vertices vertex_lat /
 *                         vertex_lon [first_vertex .. first_vertex + n_vertices), or with arg = inside = 0 outside it
 *   OC_WHERE_FILTER       an existing handle (src = oc_filter *), e.g. NOT(uncommitted deletes), built once per commit
 *   OC_WHERE_AND / OR     pops arg >= 2 values, pushes their And / Or
 *   OC_WHERE_NOT          pops one value, pushes its complement within [0, nbits)
 * A program ends with exactly one value on the stack.  Query b's outputs are byte for byte those it gets with
 * q_filters[b] = oc_filter_from_where of its program.
 * Cost: the call plans on the host (identical leaves and identical programs of the batch are evaluated once; variant and
 * range leaves are resolved to document slices by binary search), then a fixed number of launches on the call's stream:
 * one scatter for every facet leaf, one for every geo leaf, one evaluation of every program, and no synchronise.  The
 * leaf and result bitmaps live in a ctx workspace of (distinct leaves + distinct programs) x nbits / 8 bytes (a program
 * of one leaf or one FILTER takes no result bitmap), kept between calls; OC_ERR_OOM when it cannot be allocated.
 * Checks (OC_ERR_INVALID unless noted; a refused call writes nothing): a NULL store or handle; a field or variant out
 * of range, a VARIANT node on a number field or a RANGE node on a bool / string_filter field, a NaN range bound,
 * unknown flag bits; invalid coordinates, a radius that is NaN, infinite or negative, fewer than 3 or more than
 * OC_GEO_MAX_VERTICES vertices, NULL vertex arrays under a polygon; a store or handle of another ctx; a store, or a
 * handle combined with other values, whose nbits differs from oc_where.nbits (a program of one FILTER node takes the
 * handle as it is, as a q_filters entry would); an unknown op; stack underflow; a program that does not end with one value; an arity below 2; more than OC_WHERE_MAX_NODES nodes or
 * a stack deeper than OC_WHERE_MAX_DEPTH in one program; q_where together with filter, filter_bits or q_filters.
 * Entry points: those that take q_filters take q_where (a query with a program counts as filtered there); those that
 * refuse q_filters refuse q_where with the same code; a sharded call refuses it with OC_ERR_UNSUPPORTED. */
#define OC_WHERE_NONE 0u
#define OC_WHERE_VARIANT 1u
#define OC_WHERE_RANGE 2u
#define OC_WHERE_GEO_RADIUS 3u
#define OC_WHERE_GEO_POLYGON 4u
#define OC_WHERE_FILTER 5u
#define OC_WHERE_AND 6u
#define OC_WHERE_OR 7u
#define OC_WHERE_NOT 8u
#define OC_WHERE_MAX_NODES 4096u   /* nodes of one query's program                  */
#define OC_WHERE_MAX_DEPTH 32u     /* values on the stack of one program at a time  */
typedef struct oc_where_node {
    uint32_t op;             /* OC_WHERE_*                                                               */
    uint32_t field;          /* VARIANT / RANGE: the store's field                                       */
    uint32_t arg;            /* VARIANT: variant; RANGE: flags; GEO_*: inside; AND / OR: arity           */
    uint32_t first_vertex;   /* GEO_POLYGON: index into vertex_lat / vertex_lon                          */
    uint32_t n_vertices;     /* GEO_POLYGON                                                              */
    double a, b, c;          /* RANGE: lo, hi; GEO_RADIUS: lat, lon, radius_m                            */
    const void *src;         /* VARIANT / RANGE: oc_facets *; GEO_*: oc_geo_field *; FILTER: oc_filter * */
} oc_where_node;
typedef struct oc_where {
    uint64_t nbits;                   /* DocumentId space of every leaf                      */
    const uint32_t *q_node_offsets;   /* B + 1                                                */
    const oc_where_node *nodes;
    const double *vertex_lat, *vertex_lon;   /* polygon vertices (NULL when no polygon)       */
} oc_where;
/* Host only: the checks above over queries [0, n_queries), as oc_facets_check.  OC_OK or the code a search would give. */
int oc_where_check(const oc_where *w, uint32_t n_queries);
/* One query's program as an ordinary handle over [0, w->nbits), in one call with one synchronise. */
int oc_filter_from_where(oc_ctx *ctx, const oc_where *w, uint32_t query, oc_filter **out);

/* out_counts: n_queries x n_reqs.  emb / str as for oc_search (the mode decides which are needed). */
int oc_search_facets(oc_ctx *ctx, oc_emb *emb, oc_str *str, oc_facets *facets, const oc_search_params *p,
                     const oc_facet_req *reqs, uint32_t n_reqs, uint64_t *out_counts);

/* ---- groups over the score map ------------------------------------------------------------------
 * GroupContext::execute (read/index/group.rs) + sort_groups (read/sort.rs:129-230, the branch without sort_by).
 * A group is one combination of variants, one variant per listed field: the Cartesian product of the fields'
 * variants (generate_group_combinations), numbered mixed-radix over `fields` in the order given, the last field
 * varying fastest; n_groups = the product of the fields' variant counts.  Variant index: for a bool or string_filter
 * field the index it was registered with in oc_facets_add_field; for a number field the rank of its distinct value
 * in ascending order (values equal under == are one value).  Every combination is a group, also when no document
 * holds it.  A document listed under several variants of a field belongs to every matching group; ids >= the
 * facets' nbits are ignored.  Built once on the host from the fields' device lists (setup, not the hot path) and
 * kept on the device as one CSR of the groups, document ids ascending inside a group.  The handle does not refer to
 * `facets` afterwards.  OC_ERR_UNSUPPORTED: more than 2^20 groups, or a group of more than 2^32 - 2 documents. */
typedef struct oc_group_by oc_group_by;
int oc_group_by_create(oc_facets *facets, const uint32_t *fields, uint32_t n_fields, oc_group_by **out,
                       uint64_t *out_n_groups);
void oc_group_by_destroy(oc_group_by *g);
/* Hits and count exactly as oc_search with the same p; for query q and group g the top max_results documents of
 * {d in group g : d is a key of q's score map}, by final score descending, ties by ascending document id, NaN scores
 * dropped.  The score map is the one the hits come from: where-filter applied, uncommitted deletes excluded, OMC
 * multipliers applied.  max_results in [0, OC_MAX_TOPK] (0: every group present and empty).
 * p->limit == 0 is accepted here (not by oc_search): the hit arrays (out_doc_ids, out_scores, out_n; may be NULL) are
 * not written, the vector stage gets depth 0 (limit_hint = 0: no vector launch), so a hybrid score map is the fulltext
 * map alone and a vector-mode map is empty; out_count is written.
 * out_group_doc_ids / out_group_scores: B x n_groups x max_results, best first; out_group_n: B x n_groups.
 * Workspace: B x ceil(rows / 8192) x 8192 x 4 bytes of per-row scores on the device (1 GiB at B = 256 over 1M
 * string rows), OC_ERR_OOM when it cannot be allocated: pass smaller batches.  B <= 65535.
 * OC_ERR_UNSUPPORTED: p->sharded (hybrid normalisation and the vector set are global across shards),
 * max_results > OC_MAX_TOPK.  OC_ERR_INVALID: a handle of another ctx.  A failed call writes nothing.
 * Multi-index collections: run each index with limit' = limit + offset, vector_limit = limit as for oc_search, and
 * merge the group arrays with oc_merge_results over n_queries = B x n_groups, limit' = max_results. */
int oc_search_groups(oc_ctx *ctx, oc_emb *emb, oc_str *str, oc_group_by *groups, const oc_search_params *p,
                     uint32_t max_results, uint64_t *out_doc_ids, float *out_scores, uint32_t *out_n, uint64_t *out_count,
                     uint64_t *out_group_doc_ids, float *out_group_scores, uint32_t *out_group_n);

/* ---- multi-index collections ---------------------------------------------------------------------
 * search_on_indexes runs every index of a collection into ONE score map (read/search.rs:304-338,
 * token_score.rs:472-499): document ids are unique per collection, so the per-index maps are disjoint; hybrid
 * normalisation is per index; count = sum of the per-index counts; then one top_n(limit+offset) and
 * skip(offset).take(limit) (search.rs:482-498).  The caller runs oc_search once per index with
 * limit' = limit+offset, offset' = 0, vector_limit = limit and merges here (host; k sorted lists of <= limit'
 * entries).  in_stride = limit' (row stride of the per-index arrays).  Ties: ascending document id. */
int oc_merge_results(uint32_t n_indexes, uint32_t n_queries, uint32_t limit, uint32_t offset, uint32_t in_stride,
                     const uint64_t *const *doc_ids, const float *const *scores, const uint32_t *const *n,
                     const uint64_t *const *counts, uint64_t *out_doc_ids /* B x limit */, float *out_scores,
                     uint32_t *out_n, uint64_t *out_count);

/* ---- pin rules (promoted documents) ----------------------------------------------------------------
 * Search::execute collects the consequences of the pin rules that match the query (read/search.rs:127-133,
 * extract_pin_rules :257-281); sort_token_scores / sort_groups then splice their promote items into the ranking
 * (apply_pin_rules_internal, read/sort.rs:285-391).  Rule matching stays on the host; per query the caller passes the
 * promote items of the matched consequences, concatenated in the order extract_pin_rules leaves them.  Query q's items
 * are [q_pin_offsets[q], q_pin_offsets[q+1]) of doc_ids / positions (and of the per-item outputs).  A query is ACTIVE
 * when it has at least one item and apply != 0.  Deliberate deviation: a matched consequence with an empty promote list
 * doubles top_count in the reference; here it is the same as no consequence.
 * Active query, flat hits: take the top 2 x (limit + offset) of the score map (score desc, ties by ascending document id,
 * NaN dropped); remove every document the query promotes; insert the items, stably sorted by position, one after the
 * other at min(position, current length) with the document's score-map value (NaN stays NaN), or 0.0 when it is not a
 * key of the map (no match, filtered out, deleted, under the threshold, in no store); then skip(offset).take(limit).
 * So of equal positions the later item ends up in front, and a document promoted twice is inserted twice.  count is
 * unchanged (promoted non-matching documents are not counted) and the vector stage keeps depth limit.  A query that is
 * not active gets exactly oc_search's hits.  A promoted id with no stored document is dropped later by the caller's
 * document fetch, as in search.rs:181-200. */
typedef struct {
    const uint32_t *q_pin_offsets;   /* B+1, monotone                                                      */
    const uint64_t *doc_ids;         /* PromoteItem.doc_id of each item                                    */
    const uint32_t *positions;       /* PromoteItem.position                                               */
    int apply;                       /* 0: hits exactly as oc_search (no doubling, no splice): only the per-item
                                        outputs are computed — the per-index call of a multi-index search   */
} oc_pins;
/* As oc_search, plus per item its score-map value (out_pin_scores, 0.0 when not a key) and whether the document is a
 * key of the score map (out_pin_present, 1 / 0); both may be NULL.  pins may be NULL (no item).
 * OC_ERR_UNSUPPORTED: p->sharded (scores and hybrid normalisation are global), an active query with
 * 2 x (limit + offset) > OC_MAX_TOPK, a query with more than OC_MAX_TOPK items.  OC_ERR_INVALID: q_pin_offsets not
 * monotone, a handle of another ctx.  A failed call writes nothing. */
int oc_search_pinned(oc_ctx *ctx, oc_emb *emb, oc_str *str, const oc_search_params *p, const oc_pins *pins,
                     uint64_t *out_doc_ids, float *out_scores, uint32_t *out_n, uint64_t *out_count,
                     float *out_pin_scores, uint8_t *out_pin_present);
/* oc_search_groups with pins (sort_groups + apply_pin_rules_to_group, read/sort.rs:129-230, 377-391).  The flat hits
 * follow oc_search_pinned.  For an active query every group takes its top 2 x max_results, keeps the items whose
 * document is a member of the group (the group's documents, whether or not they are keys of the score map), splices
 * them as above and is NOT truncated afterwards: up to 2 x max_results + the query's member items.  A query that is not
 * active keeps exactly oc_search_groups' top max_results.  out_group_doc_ids / out_group_scores:
 * B x n_groups x group_stride; out_group_n: B x n_groups.  group_stride >= 2 x max_results + the most items of one query
 * when some query is active, else >= max_results (OC_ERR_INVALID otherwise).  Refusals as oc_search_pinned and
 * oc_search_groups, plus OC_ERR_UNSUPPORTED for an active query with 2 x max_results > OC_MAX_TOPK.  Multi-index
 * grouped searches with pins: oc_search_indexes_ex (a promoted document's membership spans indexes). */
int oc_search_groups_pinned(oc_ctx *ctx, oc_emb *emb, oc_str *str, oc_group_by *groups, const oc_search_params *p,
                            uint32_t max_results, const oc_pins *pins, uint32_t group_stride, uint64_t *out_doc_ids,
                            float *out_scores, uint32_t *out_n, uint64_t *out_count, uint64_t *out_group_doc_ids,
                            float *out_group_scores, uint32_t *out_group_n);
/* The multi-index union with pins (host, no device).  Run every index with oc_search_pinned, limit' = 2 x (limit +
 * offset), offset' = 0, vector_limit = limit, apply = 0, and pass its hit lists (in_stride = limit'), counts and per-item
 * outputs.  The per-index maps are disjoint, so a promoted document takes its score from the index where it is present,
 * else 0.0.  An active query (pins->apply) gets the union's top 2 x (limit + offset), spliced, then skip/take; any
 * other query exactly oc_merge_results' answer.  OC_ERR_INVALID: in_stride < 2 x (limit + offset) while a query is
 * active, q_pin_offsets not monotone. */
int oc_merge_pinned(uint32_t n_indexes, uint32_t n_queries, uint32_t limit, uint32_t offset, uint32_t in_stride,
                    const uint64_t *const *doc_ids, const float *const *scores, const uint32_t *const *n,
                    const uint64_t *const *counts, const oc_pins *pins, const float *const *pin_scores,
                    const uint8_t *const *pin_present, uint64_t *out_doc_ids /* B x limit */, float *out_scores,
                    uint32_t *out_n, uint64_t *out_count);

/* ---- sortBy: hits and groups in the order of a number, date or bool field --------------------------
 * sort_token_scores / sort_groups with sort_by (read/sort.rs:17-46, 48-126, 147-201): the hits are the first
 * top_count keys of the query's score map in field order, each with its score-map value; top_count = limit + offset,
 * 2 x (limit + offset) for an ACTIVE pinned query (see oc_pins).  Then the pins are spliced (as oc_search_pinned) and
 * skip(offset).take(limit).  The score map ("keys") is oc_search's: fulltext matches with the where-filter, uncommitted
 * deletes and the threshold applied, plus the vector hits at depth limit; scores are final (hybrid fusion, OMC).
 *   - count is unchanged (oc_search's), and a NaN score is KEPT: unlike score order, field order has no NotNan filter.
 *   - A key with no value in the field never appears, so a page can hold fewer than min(limit, count - offset) hits.
 *   - Order: by value (a number; a date as its i64 millisecond timestamp; a bool as 0 / 1, so false first in ASC).
 * Deliberate deviations from the reference:
 *   1. equal values: ascending document id, in both orders (the reference's order inside a value batch comes from an
 *      un-vendored crate);
 *   2. a document with several values (array field) is placed once, at its first value in the requested order: the
 *      minimum for ASC, the maximum for DESC;
 *   3. always a full page: the reference's single-index path stops collecting value batches once their total size,
 *      counting documents that are not keys, reaches top_count, so its answer is a prefix of this one; its multi-index
 *      path has no such cut and behaves as this library does everywhere;
 *   4. the multi-index merge (oc_merge_sorted) compares the true values; the reference compares i32 / f32 keys and
 *      clamps dates to the i32 range, which makes its cross-index date order effectively index order;
 *   5. as oc_pins: a matched consequence with an empty promote list does not double top_count. */
typedef struct oc_sort_field oc_sort_field;
/* One (document, value) entry per value: documents may repeat (multi-valued fields).  A bool is 0 / 1, a date its
 * millisecond timestamp; integers beyond 2^53 do not round-trip through the double and are not representable here.
 * Ids >= nbits are ignored.  OC_ERR_INVALID: a NaN value, nbits == 0 or >= 2^32 - 1; OC_ERR_UNSUPPORTED: 2^31 - 1
 * entries or more.  Built on the device under the ctx lock, on the ctx stream (radix sorts and a scan, deterministic):
 * per order the device holds the documents in rank order (8 B each) and a rank per document id (4 x nbits bytes),
 * plus a rank -> string row map rebuilt on the first sorted search after each oc_str_commit; the host keeps a copy of
 * the ranks and of each rank's value (+0.0 for a -0.0 entry).  Workspace, freed before the call returns: about 40 B
 * per entry (16 B more for the upload of oc_sort_field_create's entries), 4 B per document id and the CUB storage.
 * The handle is immutable: a changed field means a new handle. */
int oc_sort_field_create(oc_ctx *ctx, uint64_t nbits, uint64_t n, const uint64_t *doc_ids, const double *values,
                         oc_sort_field **out);
/* The sort field of one field of the facet store's published version, built on the device from the field's device
 * arrays (nothing is read back to the host first) by the same build as oc_sort_field_create, over nbits = the
 * version's.  A number or date field: variant_values NULL, each entry's value is its field value.  A bool or
 * string_filter field: variant_values holds one value per variant (a bool field {1.0, 0.0}: variant 0 is true), and a
 * document with several variants is placed by the rules above.  It runs under the ctx lock, so it reads one whole
 * published version even while an oc_facets_commit_ex of the store is in flight; the handle records that version's
 * number (oc_filter_commit_t.version, 0 before the first commit) and, like a created one, is immutable: build a new
 * one after a commit of its field.  OC_ERR_INVALID, creating nothing: a NULL argument, an unknown field,
 * variant_values NULL for a variant field or given for a number field, a NaN variant value, nbits >= 2^32 - 1. */
int oc_sort_field_from_facets(oc_facets *f, uint32_t field, const double *variant_values, oc_sort_field **out);
/* Read-back of one order (OC_SORT_ASC / OC_SORT_DESC): *n documents in rank order and the value each was placed by.
 * With rank_doc and rank_value NULL it returns the sizes; otherwise *n is the arrays' capacity on entry.  nbits and
 * facets_version (oc_sort_field_from_facets' version, 0 for a created handle) may be NULL. */
int oc_sort_field_read(const oc_sort_field *f, int order, uint64_t *nbits, uint64_t *n, uint64_t *rank_doc, double *rank_value,
                       uint64_t *facets_version);
void oc_sort_field_destroy(oc_sort_field *f);
#define OC_SORT_ASC 0
#define OC_SORT_DESC 1
typedef struct {
    const oc_sort_field *field;
    int order;                       /* OC_SORT_ASC (the reference's default) or OC_SORT_DESC */
} oc_sort;
/* oc_search_pinned in field order.  out_doc_ids / out_scores / out_sort_values: B x limit; a hit's sort value is the
 * value it was placed by, NaN for a promoted item (placed by its position); out_sort_values may be NULL.  out_n: hits written; out_count:
 * oc_search's count.  pins may be NULL; out_pin_scores / out_pin_present as in oc_search_pinned (may be NULL).
 * OC_ERR_UNSUPPORTED: p->sharded, limit + offset > OC_MAX_TOPK, an active query with 2 x (limit + offset) >
 * OC_MAX_TOPK.  OC_ERR_INVALID: a bad order, a NULL sort or field, a handle of another ctx.  A failed call writes
 * nothing. */
int oc_search_sorted(oc_ctx *ctx, oc_emb *emb, oc_str *str, const oc_search_params *p, const oc_sort *sort,
                     const oc_pins *pins, uint64_t *out_doc_ids, float *out_scores, double *out_sort_values,
                     uint32_t *out_n, uint64_t *out_count, float *out_pin_scores, uint8_t *out_pin_present);
/* One batch in which every query has its own sort, its own pins and (q_filters) its own where-filter: the batched form
 * of Search::execute with a per-request sort_by and pin rules.  Query b's outputs (hits, scores, n, count, sort values
 * and its items' pin scores / present flags) are exactly what it gets alone (B = 1) with its own filter and items:
 *   - q_sorts[b].field != NULL: oc_search_sorted with q_sorts[b];
 *   - q_sorts[b].field == NULL: oc_search_pinned (score order); its sort values are NaN, past out_n 0.0.
 * So a batch whose entries all hold one sort, without q_filters, equals oc_search_sorted, and a batch of NULL fields
 * equals oc_search_pinned.  q_sorts: B entries.  Outputs as oc_search_sorted; pins may be NULL.
 * OC_ERR_INVALID: q_sorts NULL, a bad order in an entry with a field, a sort field, filter or store of another ctx,
 * q_filters together with filter / filter_bits, q_pin_offsets not monotone.  OC_ERR_UNSUPPORTED: p->sharded, and the
 * limit + offset limits of oc_search_sorted / oc_search_pinned.  A failed call writes nothing. */
int oc_search_q_sorted(oc_ctx *ctx, oc_emb *emb, oc_str *str, const oc_search_params *p, const oc_sort *q_sorts,
                       const oc_pins *pins, uint64_t *out_doc_ids, float *out_scores, double *out_sort_values,
                       uint32_t *out_n, uint64_t *out_count, float *out_pin_scores, uint8_t *out_pin_present);
/* oc_search_groups_pinned in field order: per group the first max_results members that are keys, in field order (2 x
 * max_results for an active query), with their score-map values (NaN kept), members with no value skipped; then the
 * group's member items are spliced as in oc_search_groups_pinned.  The flat hits follow oc_search_sorted (not written
 * when p->limit == 0).  group_stride follows oc_search_groups_pinned.  out_group_sort_values (B x n_groups x
 * group_stride) may be NULL.  Refusals as oc_search_sorted and oc_search_groups_pinned.  Multi-index grouped sorting
 * without pins: oc_merge_sorted over B x n_groups rows with limit = max_results. */
int oc_search_groups_sorted(oc_ctx *ctx, oc_emb *emb, oc_str *str, oc_group_by *groups, const oc_search_params *p,
                            uint32_t max_results, const oc_sort *sort, const oc_pins *pins, uint32_t group_stride,
                            uint64_t *out_doc_ids, float *out_scores, double *out_sort_values, uint32_t *out_n,
                            uint64_t *out_count, uint64_t *out_group_doc_ids, float *out_group_scores,
                            double *out_group_sort_values, uint32_t *out_group_n);
/* ---- per-query groups -------------------------------------------------------------------------------
 * Every request of the reference carries its own groupBy (SearchParams.group_by: properties and max_results), together
 * with its own where-filter, sortBy and pin rules.  oc_search_q_groups is the batched form: query b takes q_groups[b]
 * and its items (pins), and, with q_filters, its own filter.  Query b's outputs — hits, scores, sort values, n, count,
 * its items' pin scores / present flags, and its groups (ids, score bits, n, sort values) — are byte for byte what it
 * gets alone (B = 1, p->filter = q_filters[b], its own items) from:
 *   - groups NULL: oc_search_q_sorted with its sort (field NULL: score order);
 *   - groups, score order, no item: oc_search_groups(max_results);
 *   - groups, score order, items: oc_search_groups_pinned;
 *   - groups, a sort: oc_search_groups_sorted.
 * Group layout: query b's groups are the rows [G_b, G_b + n_groups(b)) of out_group_doc_ids / out_group_scores /
 * out_group_sort_values (rows x group_stride) and out_group_n (rows), G_b = the sum of n_groups(b') over b' < b (0 for a
 * query without groups).  Entries past a row's n are 0; the group sort values of a query in score order are NaN inside
 * n.  group_stride >= 2 x max_results + its items for every ACTIVE query (see oc_pins) with groups, >= max_results for
 * any other query with groups.  out_sort_values and out_group_sort_values may be NULL; the pin outputs may be NULL.
 * p->limit == 0 is accepted when every query has groups (the hits are not written, as for oc_search_groups).
 * Workspace: B x ceil(rows / 8192) x 8192 x 4 bytes of per-row scores for the whole batch, queries without groups
 * included (as oc_search_groups); OC_ERR_OOM when it cannot be allocated: pass smaller batches.
 * Refusals (nothing written): everything the four single calls refuse — OC_ERR_INVALID: q_groups NULL, a group_by,
 * sort field, filter or store of another ctx, a bad order, group_stride below a query's need, q_pin_offsets not
 * monotone, q_filters together with filter / filter_bits, p->limit == 0 with a query without groups; OC_ERR_UNSUPPORTED:
 * p->sharded, max_results > OC_MAX_TOPK, an active query with 2 x max_results > OC_MAX_TOPK, the limit + offset limits of
 * oc_search_q_sorted — and OC_ERR_UNSUPPORTED for 2^31 or more rows. */
typedef struct {
    const oc_group_by *groups;       /* NULL: this query has no groups                          */
    uint32_t max_results;            /* per query, <= OC_MAX_TOPK                               */
    oc_sort sort;                    /* field NULL: score order                                 */
} oc_group_req;
uint64_t oc_group_by_n_groups(const oc_group_by *g);   /* its n_groups (0 for NULL): lays out the group rows */
int oc_search_q_groups(oc_ctx *ctx, oc_emb *emb, oc_str *str, const oc_search_params *p, const oc_group_req *q_groups,
                       const oc_pins *pins, uint32_t group_stride, uint64_t *out_doc_ids, float *out_scores,
                       double *out_sort_values, uint32_t *out_n, uint64_t *out_count, float *out_pin_scores,
                       uint8_t *out_pin_present, uint64_t *out_group_doc_ids, float *out_group_scores,
                       double *out_group_sort_values, uint32_t *out_group_n);
/* ---- per-query facets --------------------------------------------------------------------------------
 * oc_search_q_groups with each query's own facets (SearchParams.facets), in the same call.  facets: one store for the
 * batch.  Query b's requests are facet_reqs[q_facet_offsets[b] .. q_facet_offsets[b + 1]) (an empty range: no facets);
 * out_facet_counts has q_facet_offsets[B] entries, aligned with facet_reqs (entries before q_facet_offsets[0] are not
 * written).  A request's kind follows its field: a variant of a bool / string_filter field, a range [from, to] of a
 * number field.  q_groups may be NULL: no query has groups.  Byte for byte:
 *   - query b's hits, scores, sort values, n, count, pin outputs and group rows are what oc_search_q_groups gives the same
 *     batch without facets (and so what query b gets alone);
 *   - query b's facet counts are what oc_search_facets gives it alone: B = 1, its own requests, its filter ignored.
 * A query without a filter (no q_filters entry, no p->filter / filter_bits) counts on the matched documents of the main
 * pass.  The queries with a filter and facets are re-scored without it, as the reference does (search.rs:361-396), in
 * one more pass over just their sub-batch, without groups, sorts or pins.  p->limit == 0 is accepted when every query
 * has groups or facets: the hits are not written, and both passes run the vector stage at depth 0 (limit_hint = limit).
 * Refusals (nothing written): everything oc_search_q_groups refuses; OC_ERR_INVALID: facets of another ctx, NULL
 * facets / q_facet_offsets, q_facet_offsets not monotone, an unknown field or variant, a NaN bound (oc_facets_check);
 * OC_ERR_UNSUPPORTED: p->sharded. */
int oc_facets_check(const oc_facets *f, const oc_facet_req *reqs, uint32_t n);   /* host only: OC_OK or OC_ERR_INVALID */
int oc_search_q_facets(oc_ctx *ctx, oc_emb *emb, oc_str *str, const oc_search_params *p, const oc_group_req *q_groups,
                       const oc_pins *pins, uint32_t group_stride, oc_facets *facets, const uint32_t *q_facet_offsets /* B+1 */,
                       const oc_facet_req *facet_reqs, uint64_t *out_doc_ids, float *out_scores, double *out_sort_values,
                       uint32_t *out_n, uint64_t *out_count, float *out_pin_scores, uint8_t *out_pin_present,
                       uint64_t *out_group_doc_ids, float *out_group_scores, double *out_group_sort_values,
                       uint32_t *out_group_n, uint64_t *out_facet_counts);
/* The multi-index union in field order (host, no device; MergeSortedIterator, read/sort.rs:491-559).  Run every index
 * with oc_search_sorted, limit' = limit + offset (2 x (limit + offset) when pins apply, and then apply = 0),
 * offset' = 0, vector_limit = limit, and pass its hits, sort values (in_stride = limit'), counts and per-item
 * outputs.  The lists are merged by sort value in `order`; on equal values the index listed first wins.  count = the
 * sum of the counts.  pins may be NULL; an active query is spliced as in oc_merge_pinned (a promoted item's sort
 * value is NaN).  OC_ERR_INVALID: a bad order, n > in_stride, in_stride < 2 x (limit + offset) while a query is
 * active, q_pin_offsets not monotone.  A failed call writes nothing. */
int oc_merge_sorted(uint32_t n_indexes, uint32_t n_queries, uint32_t limit, uint32_t offset, uint32_t in_stride,
                    int order, const uint64_t *const *doc_ids, const float *const *scores,
                    const double *const *sort_values, const uint32_t *const *n, const uint64_t *const *counts,
                    const oc_pins *pins, const float *const *pin_scores, const uint8_t *const *pin_present,
                    uint64_t *out_doc_ids /* B x limit */, float *out_scores, double *out_sort_values,
                    uint32_t *out_n, uint64_t *out_count);

/* ---- one call over every index of a collection ------------------------------------------------------
 * search_on_indexes (read/search.rs:283-501) in one call: every index of a collection on this ctx runs into its own top
 * list on the device, and one kernel merges them (the union, the pins and the field order), so only the merged page
 * comes back.  Index i is described by ix[i]:
 *   - request fields, equal on every index (OC_ERR_INVALID otherwise): n_queries, mode, limit, offset, vector_limit (must
 *     be 0), similarity, threshold, bm25_k, bm25_b and the contents of q_params (each entry's vector_limit must be 0);
 *   - index fields, that index's own: the token arrays (term ids of its own dictionary), q_vecs, filter / filter_bits /
 *     q_filters / q_where (over its own filter fields), and omc_doc_ids / omc_mult / n_omc or omc;
 *   - q_sorts: NULL (score order for every query) or B entries, that index's sort handle.  Query b is in field order
 *     when every index's q_sorts[b].field is set and all share one order, in score order when every entry is NULL (or
 *     q_sorts NULL); any other mix is OC_ERR_INVALID.
 * pins (may be NULL) are the collection's: the items of query b and `apply`, as in oc_pins.
 * Result, byte for byte: the documented per-index recipe — index i alone through oc_search_q_sorted with limit' =
 * limit + offset (2 x (limit + offset) for an active pinned query), offset' = 0, vector_limit = limit and pins with
 * apply = 0, merged by oc_merge_results (score order, no pins), oc_merge_pinned (score order) or oc_merge_sorted
 * (field order).  With q_params, query b gets that recipe at its own (limit_b, offset_b), as it would alone.
 *   - out_doc_ids / out_scores / out_sort_values: B x limit; out_n, out_count (the sum of the indexes' counts): B.
 *   - out_sort_values (may be NULL): the value a hit was placed by; NaN for a promoted item and in score order; 0.0
 *     past out_n.
 *   - out_pin_scores / out_pin_present (may be NULL): per item, the score from the first index whose map holds the
 *     document, else 0.0, and whether one does.
 * Memory: the indexes' top lists stay in ctx workspaces (about 24 B per (index, query, list slot)); an oc_sort_field
 * used here gets a device copy of each order's rank values (8 B per ranked document), built the first time and freed
 * with the handle.  last_timing covers every index and the merge; its d2h_bytes includes the result blobs each index's
 * re-run checks read back.
 * Refusals (nothing written): OC_ERR_UNSUPPORTED: p->sharded, a per-index depth (limit' above) over OC_MAX_TOPK;
 * OC_ERR_INVALID: n_indexes 0 or above OC_MAX_INDEXES, request fields that differ, a store, filter, sort field or OMC
 * store of another ctx, and everything the per-index call or the host merge would refuse.
 * Not covered: batching in oc_batcher, sharded collections.  Indexes run one after another on the ctx stream.
 * Callers whose indexes live on different contexts keep using the host merges above.  oc_search_indexes is
 * oc_search_indexes_ex with ex = NULL and no groups or facets. */
#define OC_MAX_INDEXES 32u
typedef struct {
    oc_emb *emb;                     /* NULL: the index has no embedding field              */
    oc_str *str;                     /* NULL: no string fields                              */
    const oc_search_params *p;       /* this index's inputs                                 */
    const oc_sort *q_sorts;          /* NULL: score order for every query; or B entries     */
} oc_index_query;
int oc_search_indexes(oc_ctx *ctx, uint32_t n_indexes, const oc_index_query *ix, const oc_pins *pins,
                      uint64_t *out_doc_ids, float *out_scores, double *out_sort_values, uint32_t *out_n,
                      uint64_t *out_count, float *out_pin_scores, uint8_t *out_pin_present);
/* oc_search_indexes with groupBy and facets across the indexes (search_on_indexes with group_by and facets,
 * read/search.rs:283-501; GroupContext, read/index/group.rs:104-168; FacetContext, read/index/facet.rs:147-209).
 * Hits, counts and pin outputs are exactly oc_search_indexes' for the same inputs.  ex (NULL: no groups, no facets) has
 * n_indexes entries, index i's:
 *   - q_groups (NULL: none) and q_group_keys: B entries each; query b's local groups are those of q_groups[b] (NULL:
 *     none), and q_group_keys[b] sends local group g to collection key q_group_keys[b][g] < q_n_keys[b].  The caller
 *     builds the key maps from the group values, so the numbering of oc_group_by need not agree across indexes.
 *   - facets, facet_reqs[n_facet_reqs] and facet_slots: request r is counted on index i alone, as oc_search_q_facets
 *     counts it (a query filtered on that index is re-scored without its filter), and added to collection slot
 *     facet_slots[r].  A slot belongs to the query whose [q_facet_offsets[b], q_facet_offsets[b + 1]) holds it.
 * Groups: query b's collection group k is the union of the local groups every index maps to k; its rows are
 * [G_b, G_b + q_n_keys[b]) of out_group_doc_ids / out_group_scores / out_group_sort_values (rows x group_stride) and
 * out_group_n, G_b = the sum of q_n_keys over the queries before b.  Each row, with m = q_max_results[b]:
 *   - score order: the top m of the union, score descending, ties by ascending document, NaN dropped (oc_merge_results
 *     over the indexes' group rows, a missing source has n = 0);
 *   - field order (query b sorted on every index, as oc_search_indexes requires): oc_merge_sorted over those rows, equal
 *     values with the lower index first;
 *   - an active pinned query: the union's top 2 x m in the row's order, with the items whose document is a member of
 *     the collection group (of any source group) spliced as oc_search_groups_pinned splices them, not truncated; an
 *     item's score is the first index whose map holds it.
 * A row's sort value is the value its hit was placed by (NaN for an item and in score order); past n, entries are 0.
 * group_stride follows oc_search_q_groups (>= m, >= 2 x m + items for an active query).
 * Facets: out_facet_counts[s] for s in [q_facet_offsets[0], q_facet_offsets[B]) is the sum over the index requests
 * mapped to s; a slot no index maps to is 0.
 * Everything runs on the ctx stream under one lock: each index's group lists stay on the device (about 12 B per
 * (index, local row, list slot)), its facet counts are added on the device, and the groups and counts come back in
 * the one merged copy.  Refusals (nothing written): everything oc_search_indexes, oc_search_q_groups and
 * oc_search_q_facets refuse; OC_ERR_INVALID: a key >= q_n_keys[b], two local groups of one index with one key for one
 * query, a facet slot outside [q_facet_offsets[0], q_facet_offsets[B]), two requests of one index on one slot, facets
 * or a group_by of another ctx, NULL q_n_keys / q_max_results with groups, NULL q_facet_offsets with facet requests;
 * OC_ERR_UNSUPPORTED: 2^31 or more collection group rows. */
typedef struct {
    const oc_group_by *const *q_groups;       /* NULL: this index adds no groups; else B entries, NULL = none for query b */
    const uint32_t *const *q_group_keys;      /* B entries: n_groups(q_groups[b]) collection keys, each < q_n_keys[b]   */
    oc_facets *facets;                        /* NULL: no facet request on this index                                   */
    uint32_t n_facet_reqs;
    const oc_facet_req *facet_reqs;
    const uint32_t *facet_slots;              /* n_facet_reqs: the collection slot each count is added to               */
} oc_index_extras;
int oc_search_indexes_ex(oc_ctx *ctx, uint32_t n_indexes, const oc_index_query *ix, const oc_index_extras *ex,
                         const oc_pins *pins, const uint32_t *q_n_keys /* B, 0 = no groups */,
                         const uint32_t *q_max_results /* B */, uint32_t group_stride,
                         const uint32_t *q_facet_offsets /* B+1, may be NULL without facets */, uint64_t *out_doc_ids,
                         float *out_scores, double *out_sort_values, uint32_t *out_n, uint64_t *out_count,
                         float *out_pin_scores, uint8_t *out_pin_present, uint64_t *out_group_doc_ids,
                         float *out_group_scores, double *out_group_sort_values, uint32_t *out_group_n,
                         uint64_t *out_facet_counts);

/* ---- term dictionary and query-term resolution (host; oc_dict_resolve_q may expand typos on a device) ------
 * The step the reference performs before the posting walk: TextParser::tokenize_and_stem(term) —
 * originals, plus stems unless `exact`, [""] when nothing is left (token_score.rs:196-209) — and the
 * expansion of every token to index terms inside StringStorage's FST (string_field.rs:208-225): the exact
 * term when `exact` (tolerance Some(0), token_score.rs:240), terms within Levenshtein distance t for
 * tolerance = Some(t) (tests/fulltext_search.rs:956-1018), prefix expansion otherwise (:633-644); an
 * exactly matching term carries exact_match_boost (tests/boost_integration.rs:449-490; the reference's
 * constant lives in oramacore_fields 0.2.0 and is not visible: 2.0 is this library's default).
 * Term ids are stable: the id a term gets from oc_dict_add_terms is the id oc_str_insert / the loaded
 * posting lists use for it.  Output = the CSR arrays of oc_search_params. */
typedef struct oc_dict oc_dict;
typedef struct oc_resolved oc_resolved;
/* writes the stem of tok[0..len) into out (cap bytes) and returns its length; 0 = no stem */
typedef size_t (*oc_stem_fn)(const char *tok, size_t len, char *out, size_t cap, void *user);
typedef struct {
    const char *const *texts;   /* n_queries NUL-terminated query strings ("term" of SearchParams)        */
    uint32_t n_queries;
    int exact;                  /* exact match (types.rs "exact")                                          */
    int tolerance;              /* < 0: None => prefix expansion; t >= 0: Levenshtein <= t (bytes)         */
    const float *field_boost;   /* n_fields, NULL = 1.0 (boost: field -> f32, token_score.rs:138-147)      */
    const uint8_t *field_mask;  /* n_fields, NULL = all string fields (properties, token_score.rs:159-178) */
    float exact_match_boost;    /* <= 0: default 2.0                                                       */
} oc_resolve_params;
int oc_dict_create(uint32_t n_fields, oc_dict **out);
void oc_dict_destroy(oc_dict *d);
int oc_dict_add_terms(oc_dict *d, uint32_t field, const char *const *terms, uint32_t n, uint32_t *out_ids);
int oc_dict_lookup(oc_dict *d, uint32_t field, const char *term, uint32_t *out_id);   /* 0xffffffff = absent */
uint32_t oc_dict_size(oc_dict *d, uint32_t field);
int oc_dict_set_stemmer(oc_dict *d, oc_stem_fn fn, void *user);
/* the Snowball English (Porter2) algorithm with the oc_stem_fn signature, from csrc/stem_en.h; pinned to its published
 * sample vocabulary: oc_dict_set_stemmer(d, oc_stem_english, NULL).  The reference's own stemmer lives in the
 * un-vendored oramacore_lib::nlp::TextParser; a host that links it passes its own function instead. */
size_t oc_stem_english(const char *tok, size_t len, char *out, size_t cap, void *user);
int oc_dict_resolve(oc_dict *d, const oc_resolve_params *p, oc_resolved **out);
/* Per-query options for oc_dict_resolve_q. */
typedef struct oc_resolve_query {
    int exact;                  /* as oc_resolve_params.exact, for this query                              */
    int tolerance;              /* < 0: prefix expansion; t >= 0: Levenshtein <= t (bytes)                 */
    const float *field_boost;   /* n_fields, NULL = 1.0                                                    */
    const uint8_t *field_mask;  /* n_fields, NULL = all string fields                                      */
} oc_resolve_query;
/* oc_dict_resolve with options per query: query b's slice of the output equals oc_dict_resolve of texts[b] alone with
 * q[b]'s exact / tolerance / field_boost / field_mask and p->exact_match_boost, byte for byte (token ranges, fields,
 * ids, order, weight bits).  q NULL: every query takes p's options, and the output equals oc_dict_resolve(d, p).
 * ctx NULL: everything runs on the host.  With a ctx, every (token, field) pair of a query with tolerance >= 1 and a
 * token of at most 64 bytes is expanded on that ctx's device; tokenising, stemming and the exact, prefix and
 * tolerance-0 expansions (binary searches) stay on the host.  The ctx keeps a mirror of the dictionary (term bytes,
 * 8 B of offset and 4 B of sorted permutation per term; oc_dict_device_bytes), refreshed by the next such call after
 * oc_dict_add_terms: only new terms' bytes are uploaded, the permutation again when it changed.  The mirror of a
 * destroyed dictionary is freed by the ctx's next device resolve or by oc_shutdown; oc_dict_destroy never touches a
 * ctx.  Refusals write nothing: OC_ERR_INVALID for what oc_dict_resolve refuses, OC_ERR_UNSUPPORTED for a tolerance
 * above 8.  Device calls serialise on the ctx lock. */
int oc_dict_resolve_q(oc_dict *d, oc_ctx *ctx, const oc_resolve_params *p, const oc_resolve_query *q, oc_resolved **out);
/* device bytes of d's mirror on ctx (0: none yet, or either is NULL) */
uint64_t oc_dict_device_bytes(oc_dict *d, oc_ctx *ctx);
void oc_resolved_arrays(const oc_resolved *r, const uint32_t **q_token_offsets, const uint32_t **token_term_offsets,
                        const uint32_t **term_field, const uint32_t **term_id, const float **term_weight,
                        uint32_t *n_tokens, uint32_t *n_terms);
/* points p's query arrays (and n_queries) at r; r must outlive the oc_search call */
void oc_resolved_fill(const oc_resolved *r, oc_search_params *p);
void oc_resolved_free(oc_resolved *r);

/* ---- micro-batching front --------------------------------------------------------------
 * The reference runs one search per request task, many at a time (bin/oramacore.rs:76-79,
 * SURVEY.md §8b "Threading"); the GPU path earns its throughput on batches.  A batcher coalesces
 * concurrent single-query oc_search calls: the first submitter of a group leads it, waits up to
 * max_wait_us (or until max_batch queries are in), runs ONE oc_search for the group and scatters
 * the per-query results to the blocked callers.  Coalesced: queries with the same (mode, limit,
 * offset, similarity, threshold, bm25_k, bm25_b, vector_limit), no host bitmap (filter_bits), no q_filters, no OMC,
 * not sharded; a device filter (p->filter) is carried into the batch as that query's q_filters entry, so filtered
 * and unfiltered requests share a batch.  Any other call is passed straight to oc_search, and a p->filter of
 * another ctx is refused with OC_ERR_INVALID before it can join a batch.  p->n_queries must be 1; outputs as for
 * oc_search with B = 1.  A query with its own q_params runs directly.
 * A request may carry its where-clause as a one-query program (p->q_where, not together with p->filter): when some
 * request of a merged call has one, the call carries q_where with the requests' nodes concatenated (polygon vertices
 * copied after the previous requests' ones), a p->filter request as a one-node OC_WHERE_FILTER program and an
 * unfiltered request as an empty range; a merged call without programs carries q_filters as above.  A program the
 * library would refuse (every check of a where program, with the batcher's ctx as the ctx its stores and handles must
 * belong to) is refused with that error before the request joins a batch; programs over different nbits are not merged.
 * A merged call with programs that fails with OC_ERR_OOM (its bitmap workspace) is split in halves and re-run.
 * oc_batcher_create2 with flags OC_BATCHER_MIXED: the key drops mode, limit, offset, similarity, threshold and
 * vector_limit.  The merged call carries each request's scalars as its q_params entry (row stride = the largest
 * limit) and every caller gets its hits at its own limit, byte for byte what it gets alone.  The key keeps bm25_k,
 * bm25_b, the class (flat / grouped / faceted on one store), the OMC arrays (requests with identical omc_doc_ids,
 * omc_mult, n_omc batch; OMC no longer sends a request straight to oc_search) and two route flags: whether the query
 * has a threshold (text part), and whether its vector depth exceeds the tensor-core sweep's 128.  A request whose
 * limit + offset or vector depth the library refuses, or a flat request at limit 0, runs directly.
 * oc_batcher_create == oc_batcher_create2 with flags 0.  OC_ERR_INVALID: unknown flag bits. */
typedef struct oc_batcher oc_batcher;
#define OC_BATCHER_MIXED 1u
int oc_batcher_create(oc_ctx *ctx, oc_emb *emb, oc_str *str, uint32_t max_batch, uint32_t max_wait_us, oc_batcher **out);
int oc_batcher_create2(oc_ctx *ctx, oc_emb *emb, oc_str *str, uint32_t max_batch, uint32_t max_wait_us, uint32_t flags,
                       oc_batcher **out);
void oc_batcher_destroy(oc_batcher *b);
int oc_batcher_search(oc_batcher *b, const oc_search_params *p, uint64_t *out_doc_ids, float *out_scores,
                      uint32_t *out_n, uint64_t *out_count);
/* oc_batcher_search with a sort and pin rules: one query, its sort (NULL: score order) and its items (pins may be NULL;
 * q_pin_offsets has 2 entries).  Outputs as oc_search_q_sorted with B = 1: out_doc_ids / out_scores / out_sort_values
 * hold limit entries (out_sort_values may be NULL), out_pin_scores / out_pin_present (may be NULL) item j at
 * q_pin_offsets[0] + j.  Requests of both entry points share a
 * batch when their (mode, limit, offset, similarity, threshold, bm25_k, bm25_b, vector_limit) match; a batch with no
 * sort and no item runs as oc_search, any other as oc_search_q_sorted (the items concatenated in request order, each
 * p->filter as its q_filters entry).  A sort field of another ctx, a bad order or malformed pins are refused with
 * OC_ERR_INVALID before the request joins a batch.  A request the merged call could not take runs alone through
 * oc_search_q_sorted and gets its normal error there: one oc_batcher_search would not coalesce, items with apply = 0,
 * more than OC_MAX_TOPK items, or items with 2 x (limit + offset) > OC_MAX_TOPK. */
int oc_batcher_search_sorted(oc_batcher *b, const oc_search_params *p, const oc_sort *sort, const oc_pins *pins,
                             uint64_t *out_doc_ids, float *out_scores, double *out_sort_values, uint32_t *out_n,
                             uint64_t *out_count, float *out_pin_scores, uint8_t *out_pin_present);
/* oc_batcher_search_sorted with groupBy: one query, its oc_group_req, its items and group_stride; outputs as
 * oc_search_q_groups with B = 1 (its groups are rows [0, n_groups)).  Grouped requests batch only with grouped requests
 * of the same (mode, limit, offset, similarity, threshold, bm25_k, bm25_b, vector_limit); their handles, max_results,
 * sorts, items and filters may differ.  The batch runs as one oc_search_q_groups at the largest stride of its requests,
 * and each request's rows go back at its own group_stride.  Refused with OC_ERR_INVALID before joining a batch: a
 * group_stride below the request's need, malformed pins, a bad order, a handle of another ctx.  A request the merged
 * call would refuse (max_results > OC_MAX_TOPK, items with apply = 0, more than OC_MAX_TOPK items, items with
 * 2 x (limit + offset) or 2 x max_results > OC_MAX_TOPK, no groups at limit 0) runs alone and gets its normal error.  A merged call
 * that fails with OC_ERR_OOM (its row-score workspace) is split in halves and re-run, down to single requests. */
int oc_batcher_search_groups(oc_batcher *b, const oc_search_params *p, const oc_group_req *req, const oc_pins *pins,
                             uint32_t group_stride, uint64_t *out_doc_ids, float *out_scores, double *out_sort_values,
                             uint32_t *out_n, uint64_t *out_count, float *out_pin_scores, uint8_t *out_pin_present,
                             uint64_t *out_group_doc_ids, float *out_group_scores, double *out_group_sort_values,
                             uint32_t *out_group_n);
/* oc_batcher_search_groups with facets: one query, its facet store and n_facet_reqs requests, its oc_group_req or NULL (no
 * groups), items and group_stride; outputs as oc_search_q_facets with B = 1 (out_facet_counts: n_facet_reqs entries).
 * Faceted requests batch only with faceted requests of the same key and the same facet store; the batch runs as one
 * oc_search_q_facets with the requests concatenated in request order, and each caller gets its own counts.  Refused with
 * OC_ERR_INVALID before joining a batch: everything oc_batcher_search_groups refuses, facets of another ctx, and requests
 * oc_facets_check refuses.  A merged call that fails with OC_ERR_OOM is split in halves and re-run. */
int oc_batcher_search_faceted(oc_batcher *b, const oc_search_params *p, oc_facets *facets, const oc_facet_req *facet_reqs,
                              uint32_t n_facet_reqs, const oc_group_req *req, const oc_pins *pins, uint32_t group_stride,
                              uint64_t *out_doc_ids, float *out_scores, double *out_sort_values, uint32_t *out_n,
                              uint64_t *out_count, float *out_pin_scores, uint8_t *out_pin_present,
                              uint64_t *out_group_doc_ids, float *out_group_scores, double *out_group_sort_values,
                              uint32_t *out_group_n, uint64_t *out_facet_counts);
/* queries that went through a coalesced batch (grouped ones included) / number of batches / calls passed straight
 * through */
int oc_batcher_stats(oc_batcher *b, uint64_t *n_queries, uint64_t *n_batches, uint64_t *n_direct);

/* ---- pinned host buffers (optional) ----------------------------------------------------------
 * Query vectors handed to oc_search from memory obtained here (or otherwise page-locked) are
 * DMA'd straight from the caller's buffer; pageable buffers are staged through a pinned blob. */
int oc_pinned_alloc(size_t bytes, void **out);
void oc_pinned_free(void *p);

/* ---- measurement ------------------------------------------------------------------------
 * CUDA-event timings (ms, on the ctx stream) of the last oc_search / oc_emb_search on this
 * ctx, and launch counts. */
typedef struct {
    float h2d_ms;        /* query / term / filter upload                                   */
    float device_ms;     /* all kernels of the call (inputs resident)                      */
    float d2h_ms;        /* result download                                                */
    float scan_ms;       /* embedding scan kernel(s) only                                  */
    float bm25_ms;       /* posting-list scorer kernel(s) only                             */
    float fuse_ms;       /* merge / fusion / top-k kernel(s)                               */
    float comm_ms;       /* all-gather + cross-shard merge                                 */
    uint32_t kernel_launches;
    uint32_t scan_launches;
    uint64_t scan_bytes;     /* algorithmic bytes swept by the scan kernels (rows x stride x elem) */
    uint64_t bm25_postings;  /* postings walked by the scorer (x8 B = algorithmic bytes)    */
    uint64_t h2d_bytes, d2h_bytes;
    uint32_t scan_tensor_core;   /* 1 => the batched wgmma (fp16/tf32/bf16 select + exact re-score) scan ran */
    uint32_t scan_unproven;      /* queries whose candidate buffers overflowed in the tensor-core scan and were
                                    re-run through the exact sweep (device_ms includes that re-run)     */
    uint32_t scan_variant;       /* OC_SCAN_*: which sweep kernel served the batch                      */
    float scan_sweep_ms;         /* device time of the sweep launch(es) alone (scan_ms also holds the threshold pass) */
    float rerun_ms;              /* device time of re-running flagged queries (exact sweep + second tail), in device_ms */
    uint32_t scan_rescored;      /* rows re-scored in exact fp32 per query (batch average) by the tensor-core scan */
    uint32_t bm25_dense_items;   /* dense passes of the register-folded BM25 scorers: one per (query, tile) item with
                                    hot-term (dense) tokens, one more per re-run after a candidate-buffer overflow  */
    uint32_t bm25_dense_skipped; /* of those, items whose dense scan was replaced by a count pass: no row scored only by
                                    hot terms could reach the query's running top-n threshold                      */
} oc_timing;
#define OC_SCAN_EXACT 0          /* emb_scan_kernel: exact fp32 sweep (B < 8, limit > 32, tiny stores)          */
#define OC_SCAN_TC_TF32 1        /* emb_gemm_kernel: wgmma .tf32 on the fp32 rows, one CTA per SM and query group */
#define OC_SCAN_TC_BF16 4        /* emb_gemm_kernel on a bf16 store (wgmma .bf16)                                */
#define OC_SCAN_TC_F16 5         /* emb_gemm_kernel: wgmma .f16 on the fp16 copy of an fp32 store (OC_EMB_F16=0: tf32) */
int oc_last_timing(oc_ctx *ctx, oc_timing *out);
/* Total kernels this library has launched on ctx since oc_init. */
uint64_t oc_launch_count(oc_ctx *ctx);

#ifdef __cplusplus
}
#endif
#endif
