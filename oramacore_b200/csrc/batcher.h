// batcher.h — micro-batching front for concurrent single-query callers (host only, no CUDA).
//
// The reference runs ONE search per tokio task, many at a time (SURVEY.md §8b "Threading");
// the GPU path earns its throughput on batches.  SURVEY §8b allows "a batching queue" behind the
// boundary: threads submit one query each, the first submitter of a group becomes its leader,
// waits up to max_wait_us (or until max_batch queries are in), merges the group's query
// descriptors into ONE oc_search_params, runs it through `Exec` (oc_search in the library, a fake
// in tests/batcher_test.cpp) and scatters the per-query results back to the waiting callers.
// Only queries that can share a batch are coalesced: same (mode, limit, offset, similarity,
// threshold, bm25_k, bm25_b, vector_limit), no host bitmap (filter_bits), no q_filters, no OMC, not
// sharded; anything else runs directly.  A device filter (p->filter) is per query: the merged batch
// carries it as that query's q_filters entry, so filtered and unfiltered requests share a batch.
// Requests of submit_sorted carry a sort (or score order) and pin items of their own and share batches with plain
// requests: a batch with no sort and no item runs through `Exec` as before, any other through `SortedExec`
// (oc_search_q_sorted) with the sorts and the items' CSR merged in request order.
// Requests of submit_groups carry an oc_group_req and batch only with each other (the key's `grouped` bit): a batch runs
// through `GroupedExec` (oc_search_q_groups) at the largest need of its requests as the group stride, and each request's
// group rows go back at its own stride.  A merged call that runs out of device memory is split in halves and re-run.
// Requests of submit_faceted carry a facet store, their facet requests and optionally an oc_group_req; they batch only
// with faceted requests on the same store (the key's `faceted` bit and store) and run through `FacetedExec`
// (oc_search_q_facets) with the facet requests concatenated in request order; the counts go back to each caller.
#pragma once
#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstring>
#include <limits>
#include <mutex>
#include <vector>

#include "../../include/oramacore_b200.h"

namespace ocb {

struct BatchKey {
    int mode; uint32_t limit, offset; float similarity, threshold, k, b; uint32_t vector_limit;
    bool grouped = false, faceted = false;
    const oc_facets *facets = nullptr;   // faceted requests batch only on the same store
    bool operator==(const BatchKey &o) const {
        return mode == o.mode && limit == o.limit && offset == o.offset && vector_limit == o.vector_limit && grouped == o.grouped &&
               faceted == o.faceted && facets == o.facets &&
               memcmp(&similarity, &o.similarity, 4) == 0 &&
               memcmp(&threshold, &o.threshold, 4) == 0 && memcmp(&k, &o.k, 4) == 0 && memcmp(&b, &o.b, 4) == 0;
    }
};
inline BatchKey key_of(const oc_search_params *p) {
    return BatchKey{p->mode, p->limit, p->offset, p->similarity, p->threshold, p->bm25_k, p->bm25_b, p->vector_limit};
}
// has_emb / has_str: the stores the batcher was created with.  A call that oc_search would reject
// (unknown mode, missing store, NULL query arrays) is NOT batchable: it goes straight to the
// executor so the caller gets oc_search's normal error instead of a merge that dereferences NULL.
inline bool batchable(const oc_search_params *p, bool has_emb = true, bool has_str = true) {
    if (p->n_queries != 1 || p->filter_bits || p->q_filters || p->n_omc != 0 || p->sharded) return false;
    if (p->mode != OC_MODE_FULLTEXT && p->mode != OC_MODE_VECTOR && p->mode != OC_MODE_HYBRID) return false;
    const bool need_v = p->mode != OC_MODE_FULLTEXT, need_ft = p->mode != OC_MODE_VECTOR;
    if (need_v && (!has_emb || !p->q_vecs)) return false;
    if (need_ft) {
        if (!has_str || !p->q_token_offsets) return false;
        const uint32_t t0 = p->q_token_offsets[0], t1 = p->q_token_offsets[1];
        if (t1 < t0) return false;
        if (t1 > t0 && !p->token_term_offsets) return false;
        if (t1 > t0 && p->token_term_offsets[t1] > p->token_term_offsets[t0] && (!p->term_field || !p->term_id)) return false;
    }
    return true;
}

// The items of a one-query oc_pins (none for NULL); the library's checks of q_pin_offsets / doc_ids / positions.
inline uint32_t pin_items(const oc_pins *pins) { return pins ? pins->q_pin_offsets[1] - pins->q_pin_offsets[0] : 0u; }
// OC_OK, or OC_ERR_INVALID (with *why) for a request of submit_sorted the library would refuse for its own arguments:
// it must not join, and fail, a batch.
inline int check_sorted(const oc_sort *sort, const oc_pins *pins, const char **why) {
    if (sort && sort->field && sort->order != OC_SORT_ASC && sort->order != OC_SORT_DESC) { *why = "sort order is neither ASC nor DESC"; return OC_ERR_INVALID; }
    if (pins) {
        if (!pins->q_pin_offsets) { *why = "pins: q_pin_offsets is NULL"; return OC_ERR_INVALID; }
        if (pins->q_pin_offsets[1] < pins->q_pin_offsets[0]) { *why = "pins: q_pin_offsets is not monotone"; return OC_ERR_INVALID; }
        if (pin_items(pins) && (!pins->doc_ids || !pins->positions)) { *why = "pins: doc_ids / positions are NULL"; return OC_ERR_INVALID; }
    }
    return OC_OK;
}
// Whether a request's items can join a merged oc_search_q_sorted without failing it.  apply = 0 with items (the
// per-index call of a multi-index search) cannot share the merged apply = 1 CSR.  More than OC_MAX_TOPK items, or items
// with 2 x (limit + offset) > OC_MAX_TOPK, make the library refuse the whole call with OC_ERR_UNSUPPORTED: such a
// request runs alone and gets that error, and the requests it would have joined do not.
inline bool pins_batchable(const oc_search_params *p, const oc_pins *pins) {
    const uint32_t k = pin_items(pins);
    if (!k) return true;
    return pins->apply && k <= OC_MAX_TOPK && (uint64_t(p->limit) + p->offset) * 2 <= OC_MAX_TOPK;
}

// The group rows a request needs: 2 x max_results + its items when it is active, max_results otherwise, 0 without groups.
inline uint64_t group_need(const oc_group_req *req, const oc_pins *pins) {
    if (!req->groups) return 0;
    const uint32_t k = pins && pins->apply ? pin_items(pins) : 0u;
    return k ? 2ull * req->max_results + k : req->max_results;
}
// Whether a request of submit_groups can join a merged oc_search_q_groups without failing it (see pins_batchable).
inline bool groups_batchable(const oc_search_params *p, const oc_group_req *req, const oc_pins *pins) {
    if (!pins_batchable(p, pins)) return false;
    if (!req->groups) return p->limit > 0;
    return req->max_results <= OC_MAX_TOPK && (!pin_items(pins) || 2ull * req->max_results <= OC_MAX_TOPK);
}
// Whether a request of submit_faceted can join a merged oc_search_q_facets: as groups_batchable, except that a request
// without groups but with facets may run at limit 0.
inline bool faceted_batchable(const oc_search_params *p, const oc_group_req *req, const oc_pins *pins, uint32_t n_facets) {
    if (!req->groups && p->limit == 0 && n_facets) return pins_batchable(p, pins);
    return groups_batchable(p, req, pins);
}
// The request of a faceted query without groupBy.
inline const oc_group_req *no_groups() {
    static const oc_group_req none{nullptr, 0, oc_sort{nullptr, OC_SORT_ASC}};
    return &none;
}

struct BatchReq {
    const oc_search_params *p;
    uint64_t *docs; float *scores; uint32_t *n; uint64_t *count;
    // submit_sorted only
    const oc_sort *sort = nullptr;      // NULL or field NULL: score order
    const oc_pins *pins = nullptr;      // this query's items, NULL: none
    double *sort_values = nullptr;      // [limit]
    float *pin_scores = nullptr;        // [items], may be NULL
    uint8_t *pin_present = nullptr;
    // submit_groups only
    bool grouped = false;
    const oc_group_req *greq = nullptr;
    uint64_t n_groups = 0;              // its handle's n_groups (0 without groups)
    uint32_t group_stride = 0;
    uint64_t *g_doc = nullptr;          // [n_groups][group_stride]
    float *g_score = nullptr;
    double *g_values = nullptr;         // may be NULL
    uint32_t *g_n = nullptr;            // [n_groups]
    // submit_faceted only (also grouped)
    bool faceted = false;
    const oc_facets *facets = nullptr;
    const oc_facet_req *f_reqs = nullptr;
    uint32_t n_f = 0;
    uint64_t *f_counts = nullptr;       // [n_f]
    int rc = 0;
    bool done = false;
};

// Merged descriptors of one batch (owns the concatenated arrays the merged params point into).
struct MergedBatch {
    oc_search_params p{};
    std::vector<float> q_vecs, term_weight;
    std::vector<uint32_t> q_token_offsets, token_term_offsets, term_field, term_id;
    std::vector<uint64_t> docs, count;
    std::vector<float> scores;
    std::vector<uint32_t> n;
    std::vector<const oc_filter *> q_filters;   // [B] each query's p->filter, or empty when no query has one
    // a batch with a sort or an item: oc_search_q_sorted's arguments
    bool sorted = false;
    std::vector<oc_sort> q_sorts;               // [B]
    std::vector<uint32_t> pin_off, pin_pos;     // [B + 1], [items]
    std::vector<uint64_t> pin_doc;
    oc_pins pins{};
    std::vector<double> sort_values;            // [B][limit]
    std::vector<float> pin_scores;              // [items]
    std::vector<uint8_t> pin_present;
    // a grouped batch: oc_search_q_groups' arguments, each request's rows from g_row[i]
    bool grouped = false;
    std::vector<oc_group_req> q_groups;         // [B]
    std::vector<uint64_t> g_row;                // [B + 1]
    uint32_t stride = 0;
    std::vector<uint64_t> g_doc;                // [rows][stride]
    std::vector<float> g_score;
    std::vector<double> g_values;
    std::vector<uint32_t> g_n;                  // [rows]
    // a faceted batch (also grouped): oc_search_q_facets' requests, query i's at [f_off[i], f_off[i + 1])
    bool faceted = false;
    std::vector<uint32_t> f_off;                // [B + 1]
    std::vector<oc_facet_req> f_reqs;
    std::vector<uint64_t> f_counts;

    void build(const std::vector<BatchReq *> &reqs, uint32_t dim) {
        const oc_search_params *f = reqs[0]->p;
        const uint32_t B = (uint32_t)reqs.size();
        p = *f;
        p.n_queries = B;
        const bool has_v = f->mode != OC_MODE_FULLTEXT, has_ft = f->mode != OC_MODE_VECTOR;
        if (has_v) {
            q_vecs.resize(size_t(B) * dim);
            for (uint32_t i = 0; i < B; i++) memcpy(q_vecs.data() + size_t(i) * dim, reqs[i]->p->q_vecs, size_t(dim) * 4);
            p.q_vecs = q_vecs.data();
        }
        if (has_ft) {
            q_token_offsets.assign(1, 0u);
            token_term_offsets.assign(1, 0u);
            for (uint32_t i = 0; i < B; i++) {
                const oc_search_params *r = reqs[i]->p;
                const uint32_t t0 = r->q_token_offsets[0], t1 = r->q_token_offsets[1];
                for (uint32_t t = t0; t < t1; t++) {
                    const uint32_t e0 = r->token_term_offsets[t], e1 = r->token_term_offsets[t + 1];
                    for (uint32_t e = e0; e < e1; e++) {
                        term_field.push_back(r->term_field[e]);
                        term_id.push_back(r->term_id[e]);
                        term_weight.push_back(r->term_weight ? r->term_weight[e] : 1.0f);
                    }
                    token_term_offsets.push_back((uint32_t)term_id.size());
                }
                q_token_offsets.push_back((uint32_t)token_term_offsets.size() - 1);
            }
            p.q_token_offsets = q_token_offsets.data();
            p.token_term_offsets = token_term_offsets.data();
            // empty vectors still need non-NULL pointers for the ABI's argument checks
            static const uint32_t zero_u = 0; static const float one_f = 1.0f;
            p.term_field = term_field.empty() ? &zero_u : term_field.data();
            p.term_id = term_id.empty() ? &zero_u : term_id.data();
            p.term_weight = term_weight.empty() ? &one_f : term_weight.data();
        }
        q_filters.clear();
        p.filter = nullptr; p.q_filters = nullptr;
        for (uint32_t i = 0; i < B; i++)
            if (reqs[i]->p->filter) {
                q_filters.resize(B, nullptr);
                for (uint32_t j = 0; j < B; j++) q_filters[j] = reqs[j]->p->filter;
                p.q_filters = q_filters.data();
                break;
            }
        docs.assign(size_t(B) * f->limit, 0); scores.assign(size_t(B) * f->limit, 0.f);
        n.assign(B, 0); count.assign(B, 0);
        grouped = reqs[0]->grouped;
        sorted = grouped;
        for (uint32_t i = 0; i < B; i++) sorted = sorted || (reqs[i]->sort && reqs[i]->sort->field) || pin_items(reqs[i]->pins);
        if (!sorted) return;
        q_sorts.assign(B, oc_sort{nullptr, OC_SORT_ASC});
        pin_off.assign(1, 0u); pin_doc.clear(); pin_pos.clear();
        for (uint32_t i = 0; i < B; i++) {
            const BatchReq *r = reqs[i];
            if (r->sort) q_sorts[i] = *r->sort;
            if (const uint32_t k = pin_items(r->pins)) {
                const uint32_t o = r->pins->q_pin_offsets[0];
                pin_doc.insert(pin_doc.end(), r->pins->doc_ids + o, r->pins->doc_ids + o + k);
                pin_pos.insert(pin_pos.end(), r->pins->positions + o, r->pins->positions + o + k);
            }
            pin_off.push_back((uint32_t)pin_doc.size());
        }
        static const uint64_t zero_d = 0; static const uint32_t zero_p = 0;
        pins = oc_pins{pin_off.data(), pin_doc.empty() ? &zero_d : pin_doc.data(), pin_pos.empty() ? &zero_p : pin_pos.data(), 1};
        sort_values.assign(size_t(B) * f->limit, 0.0);
        pin_scores.assign(std::max<size_t>(pin_doc.size(), 1), 0.f);
        pin_present.assign(std::max<size_t>(pin_doc.size(), 1), 0);
        if (!grouped) return;
        q_groups.resize(B);
        g_row.assign(1, 0);
        stride = 0;
        for (uint32_t i = 0; i < B; i++) {
            q_groups[i] = *reqs[i]->greq;
            g_row.push_back(g_row.back() + reqs[i]->n_groups);
            stride = std::max<uint32_t>(stride, (uint32_t)group_need(reqs[i]->greq, reqs[i]->pins));
        }
        const size_t rows = g_row.back();
        g_doc.assign(std::max<size_t>(rows * stride, 1), 0);
        g_score.assign(std::max<size_t>(rows * stride, 1), 0.f);
        g_values.assign(std::max<size_t>(rows * stride, 1), 0.0);
        g_n.assign(std::max<size_t>(rows, 1), 0);
        faceted = reqs[0]->faceted;
        if (!faceted) return;
        f_off.assign(1, 0u); f_reqs.clear();
        for (uint32_t i = 0; i < B; i++) {
            f_reqs.insert(f_reqs.end(), reqs[i]->f_reqs, reqs[i]->f_reqs + reqs[i]->n_f);
            f_off.push_back((uint32_t)f_reqs.size());
        }
        f_counts.assign(std::max<size_t>(f_reqs.size(), 1), 0);
        if (f_reqs.empty()) f_reqs.resize(1);   // a non-NULL array for a batch without a request
    }
    void scatter(const std::vector<BatchReq *> &reqs, int rc) const {
        const uint32_t L = p.limit;
        for (size_t i = 0; i < reqs.size(); i++) {
            BatchReq *r = reqs[i];
            r->rc = rc;
            if (rc != 0) continue;
            if (L) {   // a grouped request at limit 0 gets no hits, as from a call of its own
                memcpy(r->docs, docs.data() + i * L, size_t(L) * 8);
                memcpy(r->scores, scores.data() + i * L, size_t(L) * 4);
                *r->n = n[i];
            }
            *r->count = count[i];
            if (r->sort_values) {   // a batch run as oc_search: score order, NaN as oc_search_q_sorted writes it
                if (sorted) memcpy(r->sort_values, sort_values.data() + i * L, size_t(L) * 8);
                else for (uint32_t j = 0; j < L; j++) r->sort_values[j] = j < n[i] ? std::numeric_limits<double>::quiet_NaN() : 0.0;
            }
            if (sorted)   // the caller's item j is its entry q_pin_offsets[0] + j, as in a call of its own
                for (uint32_t j = pin_off[i]; j < pin_off[i + 1]; j++) {
                    const size_t o = r->pins->q_pin_offsets[0] + (j - pin_off[i]);
                    if (r->pin_scores) r->pin_scores[o] = pin_scores[j];
                    if (r->pin_present) r->pin_present[o] = pin_present[j];
                }
            if (grouped)   // the request's rows at its own stride; past the merged stride its rows are 0, as past n
                for (uint64_t g = 0; g < r->n_groups; g++) {
                    const size_t src = (g_row[i] + g) * stride, dst = g * r->group_stride;
                    const uint32_t w = std::min(stride, r->group_stride);
                    for (uint32_t j = 0; j < r->group_stride; j++) {
                        r->g_doc[dst + j] = j < w ? g_doc[src + j] : 0;
                        r->g_score[dst + j] = j < w ? g_score[src + j] : 0.f;
                        if (r->g_values) r->g_values[dst + j] = j < w ? g_values[src + j] : 0.0;
                    }
                    r->g_n[g] = g_n[g_row[i] + g];
                }
            if (faceted)
                for (uint32_t j = f_off[i]; j < f_off[i + 1]; j++) r->f_counts[j - f_off[i]] = f_counts[j];
        }
    }
};

// The executor of a batcher that only takes submit(): it is never called.
struct NoSortedExec {
    int operator()(const oc_search_params *, const oc_sort *, const oc_pins *, uint64_t *, float *, double *, uint32_t *,
                   uint64_t *, float *, uint8_t *) const { return OC_ERR_UNSUPPORTED; }
};

// The executor of a batcher that only takes submit() / submit_sorted(): it is never called.
struct NoGroupedExec {
    int operator()(const oc_search_params *, const oc_group_req *, const oc_pins *, uint32_t, uint64_t *, float *, double *,
                   uint32_t *, uint64_t *, float *, uint8_t *, uint64_t *, float *, double *, uint32_t *) const {
        return OC_ERR_UNSUPPORTED;
    }
};

// The executor of a batcher that takes no submit_faceted(): it is never called.
struct NoFacetedExec {
    int operator()(const oc_search_params *, const oc_group_req *, const oc_pins *, uint32_t, const oc_facets *, const uint32_t *,
                   const oc_facet_req *, uint64_t *, float *, double *, uint32_t *, uint64_t *, float *, uint8_t *, uint64_t *, float *,
                   double *, uint32_t *, uint64_t *) const {
        return OC_ERR_UNSUPPORTED;
    }
    int check(const oc_facets *, const oc_facet_req *, uint32_t) const { return OC_ERR_UNSUPPORTED; }
};

// int Exec(const oc_search_params*, uint64_t* docs, float* scores, uint32_t* n, uint64_t* count)
// int SortedExec(const oc_search_params*, const oc_sort* q_sorts, const oc_pins*, uint64_t* docs, float* scores,
//                double* sort_values, uint32_t* n, uint64_t* count, float* pin_scores, uint8_t* pin_present)
// int GroupedExec(const oc_search_params*, const oc_group_req* q_groups, const oc_pins*, uint32_t group_stride,
//                 uint64_t* docs, float* scores, double* sort_values, uint32_t* n, uint64_t* count, float* pin_scores,
//                 uint8_t* pin_present, uint64_t* g_docs, float* g_scores, double* g_sort_values, uint32_t* g_n)
// int FacetedExec(const oc_search_params*, const oc_group_req* q_groups, const oc_pins*, uint32_t group_stride,
//                 const oc_facets*, const uint32_t* q_facet_offsets, const oc_facet_req*, <GroupedExec's outputs>,
//                 uint64_t* facet_counts)
//     and int FacetedExec::check(const oc_facets*, const oc_facet_req*, uint32_t n): oc_facets_check
template <class Exec, class SortedExec = NoSortedExec, class GroupedExec = NoGroupedExec, class FacetedExec = NoFacetedExec>
class Batcher {
public:
    Batcher(Exec exec, uint32_t dim, uint32_t max_batch, uint32_t max_wait_us, bool has_emb = true, bool has_str = true,
            SortedExec sexec = SortedExec(), GroupedExec gexec = GroupedExec(), FacetedExec fexec = FacetedExec())
        : exec_(exec), sexec_(sexec), gexec_(gexec), fexec_(fexec), dim_(dim), max_batch_(max_batch ? max_batch : 1), max_wait_us_(max_wait_us),
          has_emb_(has_emb), has_str_(has_str) {}

    int submit(const oc_search_params *p, uint64_t *docs, float *scores, uint32_t *n, uint64_t *count) {
        if (!batchable(p, has_emb_, has_str_) || max_batch_ == 1) {
            direct_++;
            return exec_(p, docs, scores, n, count);
        }
        BatchReq r{p, docs, scores, n, count};
        return join(r);
    }
    // One query with its sort (NULL: score order) and pin items (NULL: none); pin outputs one per item.
    int submit_sorted(const oc_search_params *p, const oc_sort *sort, const oc_pins *pins, uint64_t *docs, float *scores,
                      double *sort_values, uint32_t *n, uint64_t *count, float *pin_scores, uint8_t *pin_present) {
        const char *why = nullptr;
        if (const int rc = check_sorted(sort, pins, &why)) return rc;
        if (!batchable(p, has_emb_, has_str_) || max_batch_ == 1 || !pins_batchable(p, pins)) {
            direct_++;
            const oc_sort none{nullptr, OC_SORT_ASC};
            return sexec_(p, sort ? sort : &none, pins, docs, scores, sort_values, n, count, pin_scores, pin_present);
        }
        BatchReq r{p, docs, scores, n, count};
        r.sort = sort; r.pins = pins; r.sort_values = sort_values; r.pin_scores = pin_scores; r.pin_present = pin_present;
        return join(r);
    }
    // One query with its oc_group_req (n_groups: its handle's, 0 without groups), items and group stride; outputs as
    // oc_search_q_groups with B = 1.  OC_ERR_INVALID without joining: a stride below the request's need, a bad order,
    // malformed pins.
    int submit_groups(const oc_search_params *p, const oc_group_req *req, uint64_t n_groups, const oc_pins *pins,
                      uint32_t group_stride, uint64_t *docs, float *scores, double *sort_values, uint32_t *n, uint64_t *count,
                      float *pin_scores, uint8_t *pin_present, uint64_t *g_doc, float *g_score, double *g_values, uint32_t *g_n) {
        const char *why = nullptr;
        if (const int rc = check_sorted(&req->sort, pins, &why)) return rc;
        if (group_stride < group_need(req, pins)) return OC_ERR_INVALID;
        if (!batchable(p, has_emb_, has_str_) || max_batch_ == 1 || !groups_batchable(p, req, pins)) {
            direct_++;
            return gexec_(p, req, pins, group_stride, docs, scores, sort_values, n, count, pin_scores, pin_present, g_doc, g_score,
                          g_values, g_n);
        }
        BatchReq r{p, docs, scores, n, count};
        r.sort = &req->sort; r.pins = pins; r.sort_values = sort_values; r.pin_scores = pin_scores; r.pin_present = pin_present;
        r.grouped = true; r.greq = req; r.n_groups = req->groups ? n_groups : 0; r.group_stride = group_stride;
        r.g_doc = g_doc; r.g_score = g_score; r.g_values = g_values; r.g_n = g_n;
        return join(r);
    }
    // One query with its facet store and requests, its oc_group_req (NULL: no groups), items and group stride; outputs as
    // oc_search_q_facets with B = 1.  OC_ERR_INVALID without joining: what submit_groups refuses, and requests the
    // executor's check refuses.
    int submit_faceted(const oc_search_params *p, const oc_facets *facets, const oc_facet_req *f_reqs, uint32_t n_f,
                       const oc_group_req *req, uint64_t n_groups, const oc_pins *pins, uint32_t group_stride, uint64_t *docs,
                       float *scores, double *sort_values, uint32_t *n, uint64_t *count, float *pin_scores, uint8_t *pin_present,
                       uint64_t *g_doc, float *g_score, double *g_values, uint32_t *g_n, uint64_t *f_counts) {
        if (!req) req = no_groups();
        const char *why = nullptr;
        if (const int rc = check_sorted(&req->sort, pins, &why)) return rc;
        if (group_stride < group_need(req, pins)) return OC_ERR_INVALID;
        if (const int rc = fexec_.check(facets, f_reqs, n_f)) return rc;
        if (!batchable(p, has_emb_, has_str_) || max_batch_ == 1 || !faceted_batchable(p, req, pins, n_f)) {
            direct_++;
            const uint32_t off[2] = {0, n_f};
            return fexec_(p, req, pins, group_stride, facets, off, f_reqs, docs, scores, sort_values, n, count, pin_scores, pin_present,
                          g_doc, g_score, g_values, g_n, f_counts);
        }
        BatchReq r{p, docs, scores, n, count};
        r.sort = &req->sort; r.pins = pins; r.sort_values = sort_values; r.pin_scores = pin_scores; r.pin_present = pin_present;
        r.grouped = true; r.greq = req; r.n_groups = req->groups ? n_groups : 0; r.group_stride = group_stride;
        r.g_doc = g_doc; r.g_score = g_score; r.g_values = g_values; r.g_n = g_n;
        r.faceted = true; r.facets = facets; r.f_reqs = f_reqs; r.n_f = n_f; r.f_counts = f_counts;
        return join(r);
    }
    void stats(uint64_t *queries, uint64_t *batches, uint64_t *direct) {
        std::lock_guard<std::mutex> g(mu_);
        if (queries) *queries = queries_;
        if (batches) *batches = batches_;
        if (direct) *direct = direct_.load();
    }

private:
    int join(BatchReq &r) {
        const oc_search_params *p = r.p;
        std::unique_lock<std::mutex> lk(mu_);
        // one group collects at a time: wait while it is full or holds a different parameter tuple
        BatchKey k = key_of(p);
        k.grouped = r.grouped;
        k.faceted = r.faceted;
        k.facets = r.facets;
        cv_slot_.wait(lk, [&] { return pending_.empty() || (pending_key_ == k && pending_.size() < max_batch_); });
        if (pending_.empty()) pending_key_ = k;
        pending_.push_back(&r);
        if (!leader_active_) {
            leader_active_ = true;
            const auto deadline = std::chrono::steady_clock::now() + std::chrono::microseconds(max_wait_us_);
            while (pending_.size() < max_batch_)
                if (cv_leader_.wait_until(lk, deadline) == std::cv_status::timeout) break;
            std::vector<BatchReq *> batch;
            batch.swap(pending_);
            leader_active_ = false;          // the next arrival leads the next group while this one runs
            cv_slot_.notify_all();
            lk.unlock();
            if (r.grouped) run_grouped(batch);
            else {
                MergedBatch m;
                m.build(batch, dim_);
                const int rc = m.sorted ? sexec_(&m.p, m.q_sorts.data(), &m.pins, m.docs.data(), m.scores.data(), m.sort_values.data(),
                                                 m.n.data(), m.count.data(), m.pin_scores.data(), m.pin_present.data())
                                        : exec_(&m.p, m.docs.data(), m.scores.data(), m.n.data(), m.count.data());
                m.scatter(batch, rc);
            }
            lk.lock();
            batches_++; queries_ += batch.size();
            for (BatchReq *b : batch) b->done = true;
            cv_done_.notify_all();
        } else {
            if (pending_.size() >= max_batch_) cv_leader_.notify_one();
            cv_done_.wait(lk, [&] { return r.done; });
        }
        return r.rc;
    }
    // One merged oc_search_q_groups (oc_search_q_facets for a faceted batch); out of device memory (the row-score workspace grows with the batch), each half runs
    // on its own, down to single requests, which then get the single call's answer.
    void run_grouped(const std::vector<BatchReq *> &reqs) {
        MergedBatch m;
        m.build(reqs, dim_);
        const int rc = m.faceted
            ? fexec_(&m.p, m.q_groups.data(), &m.pins, m.stride, reqs[0]->facets, m.f_off.data(), m.f_reqs.data(), m.docs.data(),
                     m.scores.data(), m.sort_values.data(), m.n.data(), m.count.data(), m.pin_scores.data(), m.pin_present.data(),
                     m.g_doc.data(), m.g_score.data(), m.g_values.data(), m.g_n.data(), m.f_counts.data())
            : gexec_(&m.p, m.q_groups.data(), &m.pins, m.stride, m.docs.data(), m.scores.data(), m.sort_values.data(), m.n.data(),
                     m.count.data(), m.pin_scores.data(), m.pin_present.data(), m.g_doc.data(), m.g_score.data(), m.g_values.data(),
                     m.g_n.data());
        if (rc == OC_ERR_OOM && reqs.size() > 1) {
            const size_t h = reqs.size() / 2;
            run_grouped(std::vector<BatchReq *>(reqs.begin(), reqs.begin() + h));
            run_grouped(std::vector<BatchReq *>(reqs.begin() + h, reqs.end()));
            return;
        }
        m.scatter(reqs, rc);
    }

    Exec exec_;
    SortedExec sexec_;
    GroupedExec gexec_;
    FacetedExec fexec_;
    uint32_t dim_, max_batch_, max_wait_us_;
    bool has_emb_, has_str_;
    std::mutex mu_;
    std::condition_variable cv_slot_, cv_leader_, cv_done_;
    std::vector<BatchReq *> pending_;
    BatchKey pending_key_{};
    bool leader_active_ = false;
    uint64_t queries_ = 0, batches_ = 0;
    std::atomic<uint64_t> direct_{0};
};

}  // namespace ocb
