// batcher.h — micro-batching front for concurrent single-query callers (host only, no CUDA).
//
// The reference runs ONE search per tokio task, many at a time (SURVEY.md §8b "Threading"); the GPU path earns its
// throughput on batches.  Threads submit one Request each: the Call its entry point would make for it alone.  The
// first submitter of a group becomes its leader, waits up to max_wait_us (or until max_batch requests are in), merges
// the group into ONE Call, runs it through the executor (the library's entry points, a fake in
// tests/batcher_test.cpp) and scatters each request's outputs back.  A group shares the parameter tuple (mode, limit,
// offset, similarity, threshold, bm25_k, bm25_b, vector_limit), a class: flat (PLAIN and SORTED requests), GROUPED,
// or FACETED on one facet store, and the OMC store (p->omc, or none).  A merged flat call runs as PLAIN unless a request has a sort field or an item; a
// merged grouped call runs at the largest need of its requests as the group stride.  Each request's p->filter becomes
// its q_filters entry.  A request the merged call could not take (batchable and the *_batchable predicates) runs
// directly, alone; one the library would refuse for its own arguments is refused before it joins.  A merged grouped or
// faceted call that runs out of device memory is split in halves and re-run.
// Mixed batcher (OC_BATCHER_MIXED): the key drops (mode, limit, offset, similarity, threshold, vector_limit); requests
// that differ in them share a batch, each carrying its scalars as its q_params entry of the merged call, whose limit
// (the hits' row stride) is the batch's largest.  The key keeps bm25_k, bm25_b, the class, the OMC arrays (requests on
// one index share them, so they batch) and two route flags, each of which would move a whole batch to a slower kernel:
// "has a threshold" (the threshold scorer) and "vector depth above the tensor-core limit" (the exact sweep).
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

// The library entry point of a call: oc_search, oc_search_q_sorted, oc_search_q_groups, oc_search_q_facets.
enum Kind { PLAIN, SORTED, GROUPED, FACETED };

// One executor call: oc_search_q_facets' arguments, q_sorts for SORTED, and the entry point that takes them.  Each
// entry point reads the arguments it has; the rest stay NULL.
struct Call {
    Kind kind;
    const oc_search_params *p;
    uint64_t *docs; float *scores; uint32_t *n; uint64_t *count;
    double *sort_values = nullptr;
    float *pin_scores = nullptr; uint8_t *pin_present = nullptr;
    const oc_pins *pins = nullptr;
    const oc_sort *q_sorts = nullptr;         // SORTED
    const oc_group_req *q_groups = nullptr;   // GROUPED, FACETED
    uint32_t group_stride = 0;
    uint64_t *g_docs = nullptr; float *g_scores = nullptr; double *g_values = nullptr; uint32_t *g_n = nullptr;
    oc_facets *facets = nullptr;              // FACETED
    const uint32_t *q_facet_offsets = nullptr;
    const oc_facet_req *facet_reqs = nullptr;
    uint64_t *f_counts = nullptr;
};

// One caller's query: the call it makes alone (on its own arrays), its handle's n_groups and its outcome.  A FACETED
// request's q_facet_offsets point at f_off = {0, its facet requests}.
struct Request {
    Call call;
    uint64_t n_groups = 0;
    uint32_t f_off[2] = {0, 0};
    int rc = 0;
    bool done = false;
};

// The sort of a call's first query (NULL for PLAIN).
inline const oc_sort *sort_of(const Call &c) { return c.q_groups ? &c.q_groups->sort : c.q_sorts; }
inline uint32_t n_facets(const Call &c) { return c.q_facet_offsets ? c.q_facet_offsets[1] - c.q_facet_offsets[0] : 0u; }
// The sort of a SORTED request without one, and the oc_group_req of a FACETED request without groupBy.
inline const oc_sort *score_order() {
    static const oc_sort none{nullptr, OC_SORT_ASC};
    return &none;
}
inline const oc_group_req *no_groups() {
    static const oc_group_req none{nullptr, 0, oc_sort{nullptr, OC_SORT_ASC}};
    return &none;
}

// Largest vector depth the tensor-core sweep serves (emb_gemm.cuh GEMM_MAX_LIMIT): a deeper query sends the vector
// sub-batch of its call to the exact sweep.
constexpr uint32_t TC_MAX_DEPTH = 128;

struct BatchKey {
    int mode; uint32_t limit, offset; float similarity, threshold, k, b; uint32_t vector_limit;
    Kind cls;                            // PLAIN for the flat class, GROUPED or FACETED
    const oc_facets *facets;             // faceted requests batch only on the same store
    // mixed batcher: the scalars above are 0; the route flags and the OMC arrays take their place
    bool thr, deep;
    const uint64_t *omc_doc; const float *omc_mult; uint64_t n_omc;
    const oc_omc *omc;                   // both batchers: requests batch only on the same OMC store (or none)
    bool operator==(const BatchKey &o) const {
        return mode == o.mode && limit == o.limit && offset == o.offset && vector_limit == o.vector_limit && cls == o.cls &&
               facets == o.facets && memcmp(&similarity, &o.similarity, 4) == 0 && memcmp(&threshold, &o.threshold, 4) == 0 &&
               memcmp(&k, &o.k, 4) == 0 && memcmp(&b, &o.b, 4) == 0 && thr == o.thr && deep == o.deep && omc_doc == o.omc_doc &&
               omc_mult == o.omc_mult && n_omc == o.n_omc && omc == o.omc;
    }
};
// The vector depth of a query alone (0 without a vector part): vector_limit, else limit.
inline uint32_t vector_depth(const oc_search_params *p) {
    return p->mode == OC_MODE_FULLTEXT ? 0u : p->vector_limit ? p->vector_limit : p->limit;
}
inline BatchKey key_of(const Call &c, bool mixed = false) {
    const oc_search_params *p = c.p;
    const Kind cls = c.kind == SORTED ? PLAIN : c.kind;
    if (mixed)
        return BatchKey{0, 0, 0, 0.f, 0.f, p->bm25_k, p->bm25_b, 0, cls, c.facets,
                        p->mode != OC_MODE_VECTOR && p->threshold >= 0.0f, vector_depth(p) > TC_MAX_DEPTH,
                        p->n_omc ? p->omc_doc_ids : nullptr, p->n_omc ? p->omc_mult : nullptr, p->n_omc, p->omc};
    return BatchKey{p->mode, p->limit, p->offset, p->similarity, p->threshold, p->bm25_k, p->bm25_b, p->vector_limit,
                    cls, c.facets, false, false, nullptr, nullptr, 0, p->omc};
}
// has_emb / has_str: the stores the batcher was created with.  A call that oc_search would reject
// (unknown mode, missing store, NULL query arrays) is NOT batchable: it goes straight to the
// executor so the caller gets oc_search's normal error instead of a merge that dereferences NULL.
// A request with its own q_params runs directly (the merged call's q_params are the requests' scalars).  mixed: OMC
// arrays join the key instead of keeping the request out; the scalars must pass the library's bounds, which a batch
// of equal scalars would otherwise refuse for all of its requests alike.
inline bool batchable(const oc_search_params *p, bool has_emb = true, bool has_str = true, bool mixed = false) {
    if (p->n_queries != 1 || p->filter_bits || p->q_filters || p->q_params || (p->n_omc != 0 && !mixed) || p->sharded) return false;
    if (p->q_where && p->filter) return false;
    if (p->omc && p->n_omc) return false;   // refused by the library: alone, so only this request fails
    if (mixed && (uint64_t(p->limit) + p->offset > OC_MAX_TOPK || (p->limit && (p->vector_limit ? p->vector_limit : p->limit) > OC_MAX_TOPK)))
        return false;
    if (mixed && p->n_omc && (!p->omc_doc_ids || !p->omc_mult)) return false;
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
// OC_OK, or OC_ERR_INVALID (with *why) for a sort and items the library would refuse for their own arguments: such a
// request must not join, and fail, a batch.
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
// Whether a grouped or faceted request can join a merged oc_search_q_groups / oc_search_q_facets without failing it (see
// pins_batchable).  Only a request with facets (n_facets > 0) may run without groups at limit 0.
inline bool groups_batchable(const oc_search_params *p, const oc_group_req *req, const oc_pins *pins, uint32_t n_facets) {
    if (!pins_batchable(p, pins)) return false;
    if (!req->groups) return p->limit > 0 || n_facets > 0;
    return req->max_results <= OC_MAX_TOPK && (!pin_items(pins) || 2ull * req->max_results <= OC_MAX_TOPK);
}

// The merged Call of one batch and the concatenated arrays it points into.  Built in place: `call` points at members.
struct MergedBatch {
    Call call{};
    oc_search_params p{};
    // hits
    std::vector<float> q_vecs, term_weight;
    std::vector<uint32_t> q_token_offsets, token_term_offsets, term_field, term_id;
    std::vector<uint64_t> docs, count;
    std::vector<float> scores;
    std::vector<uint32_t> n;
    std::vector<const oc_filter *> q_filters;   // [B] each query's p->filter, or empty when no query has one
    // when some query has a where program: each query's program (its p->filter as one FILTER node), polygon vertices
    // copied after the previous queries' ones
    oc_where where{};
    std::vector<uint32_t> w_off;                // [B + 1]
    std::vector<oc_where_node> w_nodes;
    std::vector<double> w_lat, w_lon;
    std::vector<oc_query_params> q_params;      // [B] mixed: each query's scalars
    // sort values and items (all but PLAIN)
    std::vector<oc_sort> q_sorts;               // [B] (SORTED)
    std::vector<uint32_t> pin_off, pin_pos;     // [B + 1], [items]
    std::vector<uint64_t> pin_doc;
    oc_pins pins{};
    std::vector<double> sort_values;            // [B][limit]
    std::vector<float> pin_scores;              // [items]
    std::vector<uint8_t> pin_present;
    // groups (GROUPED, FACETED): each request's rows from g_row[i]
    std::vector<oc_group_req> q_groups;         // [B]
    std::vector<uint64_t> g_row;                // [B + 1]
    std::vector<uint64_t> g_doc;                // [rows][stride]
    std::vector<float> g_score;
    std::vector<double> g_values;
    std::vector<uint32_t> g_n;                  // [rows]
    // facets (FACETED): query i's requests at [f_off[i], f_off[i + 1])
    std::vector<uint32_t> f_off;                // [B + 1]
    std::vector<oc_facet_req> f_reqs;
    std::vector<uint64_t> f_counts;

    void build(const std::vector<Request *> &reqs, uint32_t dim, bool mixed = false) {
        const Call &f = reqs[0]->call;
        const uint32_t B = (uint32_t)reqs.size();
        Kind kind = f.kind == SORTED ? PLAIN : f.kind;
        for (const Request *r : reqs) {
            const oc_sort *s = sort_of(r->call);
            if (kind == PLAIN && ((s && s->field) || pin_items(r->call.pins))) kind = SORTED;
        }
        build_hits(reqs, dim, mixed);
        const uint32_t L = p.limit;
        call = Call{kind, &p, docs.data(), scores.data(), n.data(), count.data()};
        if (kind != PLAIN) build_pins(reqs, L);
        if (kind == SORTED) {
            q_sorts.resize(B);
            for (uint32_t i = 0; i < B; i++) q_sorts[i] = reqs[i]->call.q_sorts ? *reqs[i]->call.q_sorts : *score_order();
            call.q_sorts = q_sorts.data();
        }
        if (kind == GROUPED || kind == FACETED) build_groups(reqs);
        if (kind == FACETED) build_facets(reqs);
    }
    // mixed: every query's scalars go into q_params; the merged limit is the largest (the row stride), the vectors of
    // the queries without a vector part are zero rows (not read) and those without a text part have no token
    void build_hits(const std::vector<Request *> &reqs, uint32_t dim, bool mixed) {
        const oc_search_params *f = reqs[0]->call.p;
        const uint32_t B = (uint32_t)reqs.size();
        p = *f;
        p.n_queries = B;
        bool any_v = f->mode != OC_MODE_FULLTEXT, any_ft = f->mode != OC_MODE_VECTOR;
        if (mixed) {
            p.limit = 0;
            any_v = any_ft = false;
            for (const Request *req : reqs) {
                const oc_search_params *r = req->call.p;
                q_params.push_back(oc_query_params{r->mode, r->limit, r->offset, r->similarity, r->threshold, r->vector_limit});
                p.limit = std::max(p.limit, r->limit);
                any_v = any_v || r->mode != OC_MODE_FULLTEXT;
                any_ft = any_ft || r->mode != OC_MODE_VECTOR;
            }
            p.q_params = q_params.data();
            p.mode = any_v && any_ft ? OC_MODE_HYBRID : any_v ? OC_MODE_VECTOR : OC_MODE_FULLTEXT;
            p.q_vecs = nullptr; p.q_token_offsets = nullptr;
        }
        if (any_v) {
            q_vecs.assign(size_t(B) * dim, 0.f);
            for (uint32_t i = 0; i < B; i++)
                if (reqs[i]->call.p->mode != OC_MODE_FULLTEXT)
                    memcpy(q_vecs.data() + size_t(i) * dim, reqs[i]->call.p->q_vecs, size_t(dim) * 4);
            p.q_vecs = q_vecs.data();
        }
        if (any_ft) {
            q_token_offsets.assign(1, 0u);
            token_term_offsets.assign(1, 0u);
            for (const Request *req : reqs) {
                const oc_search_params *r = req->call.p;
                if (r->mode == OC_MODE_VECTOR) { q_token_offsets.push_back(q_token_offsets.back()); continue; }
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
        p.filter = nullptr; p.q_filters = nullptr; p.q_where = nullptr;
        if (std::any_of(reqs.begin(), reqs.end(), [](const Request *r) { return r->call.p->q_where != nullptr; })) {
            build_where(reqs);
            return;
        }
        for (const Request *r : reqs)
            if (r->call.p->filter) {
                for (const Request *q : reqs) q_filters.push_back(q->call.p->filter);
                p.q_filters = q_filters.data();
                break;
            }
        alloc_hits(B);
    }
    void alloc_hits(uint32_t B) {
        docs.assign(size_t(B) * p.limit, 0); scores.assign(size_t(B) * p.limit, 0.f);
        n.assign(B, 0); count.assign(B, 0);
    }
    // the requests' programs concatenated (nbits: the first program's; run() keeps other sizes out of one batch)
    void build_where(const std::vector<Request *> &reqs) {
        w_off.assign(1, 0u);
        bool first = true;
        for (const Request *r : reqs) {
            const oc_search_params *rp = r->call.p;
            if (const oc_where *w = rp->q_where) {
                if (first) where.nbits = w->nbits;
                first = false;
                for (uint32_t i = w->q_node_offsets[0]; i < w->q_node_offsets[1]; i++) {
                    oc_where_node nd = w->nodes[i];
                    if (nd.op == OC_WHERE_GEO_POLYGON) {
                        const uint32_t fv = nd.first_vertex;
                        nd.first_vertex = (uint32_t)w_lat.size();
                        w_lat.insert(w_lat.end(), w->vertex_lat + fv, w->vertex_lat + fv + nd.n_vertices);
                        w_lon.insert(w_lon.end(), w->vertex_lon + fv, w->vertex_lon + fv + nd.n_vertices);
                    }
                    w_nodes.push_back(nd);
                }
            } else if (rp->filter) {
                oc_where_node nd{};
                nd.op = OC_WHERE_FILTER;
                nd.src = rp->filter;
                w_nodes.push_back(nd);
            }
            w_off.push_back((uint32_t)w_nodes.size());
        }
        where.q_node_offsets = w_off.data();
        where.nodes = w_nodes.empty() ? nullptr : w_nodes.data();
        where.vertex_lat = w_lat.empty() ? nullptr : w_lat.data();
        where.vertex_lon = w_lon.empty() ? nullptr : w_lon.data();
        p.q_where = &where;
        alloc_hits((uint32_t)reqs.size());
    }
    void build_pins(const std::vector<Request *> &reqs, uint32_t L) {
        pin_off.assign(1, 0u);
        for (const Request *r : reqs) {
            const oc_pins *rp = r->call.pins;
            if (const uint32_t k = pin_items(rp)) {
                const uint32_t o = rp->q_pin_offsets[0];
                pin_doc.insert(pin_doc.end(), rp->doc_ids + o, rp->doc_ids + o + k);
                pin_pos.insert(pin_pos.end(), rp->positions + o, rp->positions + o + k);
            }
            pin_off.push_back((uint32_t)pin_doc.size());
        }
        static const uint64_t zero_d = 0; static const uint32_t zero_p = 0;
        pins = oc_pins{pin_off.data(), pin_doc.empty() ? &zero_d : pin_doc.data(), pin_pos.empty() ? &zero_p : pin_pos.data(), 1};
        sort_values.assign(reqs.size() * L, 0.0);
        pin_scores.assign(std::max<size_t>(pin_doc.size(), 1), 0.f);
        pin_present.assign(std::max<size_t>(pin_doc.size(), 1), 0);
        call.pins = &pins;
        call.sort_values = sort_values.data(); call.pin_scores = pin_scores.data(); call.pin_present = pin_present.data();
    }
    void build_groups(const std::vector<Request *> &reqs) {
        uint32_t stride = 0;
        g_row.assign(1, 0);
        for (const Request *r : reqs) {
            q_groups.push_back(*r->call.q_groups);
            g_row.push_back(g_row.back() + r->n_groups);
            stride = std::max<uint32_t>(stride, (uint32_t)group_need(r->call.q_groups, r->call.pins));
        }
        const size_t cells = std::max<size_t>(g_row.back() * stride, 1);
        g_doc.assign(cells, 0); g_score.assign(cells, 0.f); g_values.assign(cells, 0.0);
        g_n.assign(std::max<size_t>(g_row.back(), 1), 0);
        call.q_groups = q_groups.data(); call.group_stride = stride;
        call.g_docs = g_doc.data(); call.g_scores = g_score.data(); call.g_values = g_values.data(); call.g_n = g_n.data();
    }
    void build_facets(const std::vector<Request *> &reqs) {
        f_off.assign(1, 0u);
        for (const Request *r : reqs) {
            f_reqs.insert(f_reqs.end(), r->call.facet_reqs, r->call.facet_reqs + n_facets(r->call));
            f_off.push_back((uint32_t)f_reqs.size());
        }
        f_counts.assign(std::max<size_t>(f_reqs.size(), 1), 0);
        if (f_reqs.empty()) f_reqs.resize(1);   // a non-NULL array for a batch without a request
        call.facets = reqs[0]->call.facets; call.q_facet_offsets = f_off.data(); call.facet_reqs = f_reqs.data();
        call.f_counts = f_counts.data();
    }

    void scatter(const std::vector<Request *> &reqs, int rc) const {
        const uint32_t L = p.limit, S = call.group_stride;
        for (size_t i = 0; i < reqs.size(); i++) {
            reqs[i]->rc = rc;
            if (rc != 0) continue;
            const Call &o = reqs[i]->call;
            const uint32_t Li = o.p->limit;   // the request's own row: the first Li entries of its row of L (mixed: L >= Li)
            if (Li) {   // a request at limit 0 gets no hits, as from a call of its own
                memcpy(o.docs, docs.data() + i * L, size_t(Li) * 8);
                memcpy(o.scores, scores.data() + i * L, size_t(Li) * 4);
                *o.n = n[i];
            }
            *o.count = count[i];
            if (o.sort_values) {   // a batch run as oc_search: score order, NaN as oc_search_q_sorted writes it
                if (call.kind != PLAIN) memcpy(o.sort_values, sort_values.data() + i * L, size_t(Li) * 8);
                else for (uint32_t j = 0; j < Li; j++) o.sort_values[j] = j < n[i] ? std::numeric_limits<double>::quiet_NaN() : 0.0;
            }
            if (call.kind != PLAIN)   // the caller's item j is its entry q_pin_offsets[0] + j, as in a call of its own
                for (uint32_t j = pin_off[i]; j < pin_off[i + 1]; j++) {
                    const size_t d = o.pins->q_pin_offsets[0] + (j - pin_off[i]);
                    if (o.pin_scores) o.pin_scores[d] = pin_scores[j];
                    if (o.pin_present) o.pin_present[d] = pin_present[j];
                }
            if (call.q_groups)   // the request's rows at its own stride; past the merged stride its rows are 0, as past n
                for (uint64_t g = 0; g < reqs[i]->n_groups; g++) {
                    const size_t src = (g_row[i] + g) * S, dst = g * o.group_stride;
                    const uint32_t w = std::min(S, o.group_stride);
                    for (uint32_t j = 0; j < o.group_stride; j++) {
                        o.g_docs[dst + j] = j < w ? g_doc[src + j] : 0;
                        o.g_scores[dst + j] = j < w ? g_score[src + j] : 0.f;
                        if (o.g_values) o.g_values[dst + j] = j < w ? g_values[src + j] : 0.0;
                    }
                    o.g_n[g] = g_n[g_row[i] + g];
                }
            if (call.kind == FACETED)
                for (uint32_t j = f_off[i]; j < f_off[i + 1]; j++) o.f_counts[j - f_off[i]] = f_counts[j];
        }
    }
};

// Exec: int operator()(const Call &), the call's entry point; int check(const oc_facets *, const oc_facet_req *,
// uint32_t n), oc_facets_check.
template <class Exec>
class Batcher {
public:
    Batcher(Exec exec, uint32_t dim, uint32_t max_batch, uint32_t max_wait_us, bool has_emb = true, bool has_str = true,
            bool mixed = false)
        : exec_(exec), dim_(dim), max_batch_(max_batch ? max_batch : 1), max_wait_us_(max_wait_us), has_emb_(has_emb),
          has_str_(has_str), mixed_(mixed) {}

    // Runs r (n_groups set for a grouped or faceted request) directly or in a batch and returns its code.  A request
    // the library would refuse for its own arguments gets OC_ERR_INVALID (with *why; a refusal of the facet check sets
    // no *why) and never reaches the executor.
    int submit(Request &r, const char **why) {
        const Call &c = r.call;
        if (const int rc = check_sorted(sort_of(c), c.pins, why)) return rc;
        if (c.q_groups && c.group_stride < group_need(c.q_groups, c.pins)) {
            *why = "group_stride is below the request's need";
            return OC_ERR_INVALID;
        }
        if (c.kind == FACETED)
            if (const int rc = exec_.check(c.facets, c.facet_reqs, n_facets(c))) return rc;
        bool merge = max_batch_ > 1 && batchable(c.p, has_emb_, has_str_, mixed_);
        // mixed: a flat request at limit 0 would make the library refuse the merged call of every request with it
        if (mixed_ && !c.q_groups && c.p->limit == 0) merge = false;
        if (c.kind == SORTED) merge = merge && pins_batchable(c.p, c.pins);
        if (c.q_groups) merge = merge && groups_batchable(c.p, c.q_groups, c.pins, n_facets(c));
        if (!merge) {
            direct_++;
            return exec_(c);
        }
        return join(r);
    }
    void stats(uint64_t *queries, uint64_t *batches, uint64_t *direct) {
        std::lock_guard<std::mutex> g(mu_);
        if (queries) *queries = queries_;
        if (batches) *batches = batches_;
        if (direct) *direct = direct_.load();
    }

private:
    int join(Request &r) {
        std::unique_lock<std::mutex> lk(mu_);
        // one group collects at a time: wait while it is full or holds a different key
        const BatchKey k = key_of(r.call, mixed_);
        cv_slot_.wait(lk, [&] { return pending_.empty() || (pending_key_ == k && pending_.size() < max_batch_); });
        if (pending_.empty()) pending_key_ = k;
        pending_.push_back(&r);
        if (!leader_active_) {
            leader_active_ = true;
            const auto deadline = std::chrono::steady_clock::now() + std::chrono::microseconds(max_wait_us_);
            while (pending_.size() < max_batch_)
                if (cv_leader_.wait_until(lk, deadline) == std::cv_status::timeout) break;
            std::vector<Request *> batch;
            batch.swap(pending_);
            leader_active_ = false;          // the next arrival leads the next group while this one runs
            cv_slot_.notify_all();
            lk.unlock();
            run(batch);
            lk.lock();
            batches_++; queries_ += batch.size();
            for (Request *b : batch) b->done = true;
            cv_done_.notify_all();
        } else {
            if (pending_.size() >= max_batch_) cv_leader_.notify_one();
            cv_done_.wait(lk, [&] { return r.done; });
        }
        return r.rc;
    }
    // One merged call.  A grouped or faceted one, or one with where programs, that runs out of device memory (the
    // row-score and bitmap workspaces grow with the batch) is split in halves, down to single requests, which then get
    // the single call's answer.  Programs over different DocumentId spaces cannot share a call: such a batch runs one
    // request per call.
    void run(const std::vector<Request *> &reqs) {
        const oc_where *w0 = nullptr;
        for (const Request *r : reqs) {
            const oc_where *w = r->call.p->q_where;
            if (!w) continue;
            if (w0 && w->nbits != w0->nbits && reqs.size() > 1) {
                for (Request *q : reqs) run(std::vector<Request *>{q});
                return;
            }
            w0 = w0 ? w0 : w;
        }
        MergedBatch m;
        m.build(reqs, dim_, mixed_);
        const int rc = exec_(m.call);
        if (rc == OC_ERR_OOM && (m.call.q_groups || m.p.q_where) && reqs.size() > 1) {
            const size_t h = reqs.size() / 2;
            run(std::vector<Request *>(reqs.begin(), reqs.begin() + h));
            run(std::vector<Request *>(reqs.begin() + h, reqs.end()));
            return;
        }
        m.scatter(reqs, rc);
    }

    Exec exec_;
    uint32_t dim_, max_batch_, max_wait_us_;
    bool has_emb_, has_str_, mixed_;
    std::mutex mu_;
    std::condition_variable cv_slot_, cv_leader_, cv_done_;
    std::vector<Request *> pending_;
    BatchKey pending_key_{};
    bool leader_active_ = false;
    uint64_t queries_ = 0, batches_ = 0;
    std::atomic<uint64_t> direct_{0};
};

}  // namespace ocb
