// Host-logic test of the micro-batching queue (oramacore_b200/csrc/batcher.h) with one fake executor.  Every request
// carries its id (the last component of its query vector) and ocb::Request; what it submitted is described once, in
// g_desc[id].  The fake checks each query of each call against its description, answers with values derived from the
// query's own arguments and description, and refuses what the library refuses for the sizes.  Each scenario submits
// from many threads and checks that every caller gets exactly its own answer, that requests were coalesced, and what
// reached the executor.  Run one scenario per process: batcher_test plain | qfilters | sorted | groups | facets.
// Built and run by tests/test_batcher_host.py (g++, no CUDA).
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <functional>
#include <random>
#include <thread>
#include <vector>

#include "../oramacore_b200/csrc/batcher.h"

using ocb::Kind;
static const uint32_t DIM = 8, BAD_FIELD = 99;
static const int MAX_IDS = 4000, N_HANDLES = 7, N_FIELDS = 3, N_GB = 3, N_STORES = 2;
static const uint64_t GB_GROUPS[N_GB] = {1, 3, 7};
static char g_handles[N_HANDLES], g_fields[N_FIELDS], g_gb[N_GB], g_st[N_STORES];   // fake handles: only their addresses are used
static const oc_filter *handle(int i) { return reinterpret_cast<const oc_filter *>(&g_handles[i]); }
static const oc_sort_field *field(int i) { return reinterpret_cast<const oc_sort_field *>(&g_fields[i]); }
static const oc_group_by *gb(int i) { return reinterpret_cast<const oc_group_by *>(&g_gb[i]); }
static oc_facets *store(int i) { return reinterpret_cast<oc_facets *>(&g_st[i]); }
template <class T> static int index_of(const T *h, const char *base, int n) {
    for (int i = 0; i < n; i++) if (reinterpret_cast<const char *>(h) == base + i) return i;
    return -2;
}

// What request `id` submitted.
struct Desc {
    Kind kind = ocb::PLAIN;
    bool refused = false;            // refused before it reaches the executor
    int filter = -1;                 // its device filter; 100: a host bitmap, -1: none
    int field = -1, order = 0;       // its sort; -1: score order
    uint32_t k = 0, apply = 1;       // its items
    int gb = -1;                     // its groupBy handle; -1: none
    uint32_t m = 0, stride = 0;      // max_results, group stride
    int store = -1;                  // its facet store
    uint32_t nf = 0;                 // its facet requests
};
static Desc g_desc[MAX_IDS];
static uint32_t g_oom_above = ~0u;   // a merged grouped / faceted call of more queries runs out of device memory

static uint32_t need_of(const Desc &d) { return d.gb < 0 ? 0 : d.k && d.apply ? 2 * d.m + d.k : d.m; }
static uint64_t n_groups_of(const Desc &d) { return d.gb < 0 ? 0 : GB_GROUPS[d.gb]; }
// row g of request id has (id + g) % (need + 1) entries
static uint32_t n_of(uint32_t id, uint64_t g) { return uint32_t((id + g) % (need_of(g_desc[id]) + 1)); }
static uint64_t doc_of(uint32_t id, uint64_t g, uint32_t j) { return uint64_t(id) * 100000 + g * 100 + j + 1; }
static uint32_t facet_field(uint32_t id, uint32_t j) { return g_desc[id].refused && j == 0 ? BAD_FIELD : (id + j) % 7; }
static uint64_t facet_count(uint32_t id, uint32_t j) { return uint64_t(id) * 1000 + j + 1; }
static double sort_value(int f, int order) { return f < 0 ? std::nan("") : double(2 * f + order); }

// Answers of the fake: hits from the query's vector and tokens, scores from its filter.
static long long signature(const oc_search_params *p, uint32_t i) {
    long long sig = 0;
    if (p->mode != OC_MODE_FULLTEXT) sig += (long long)llround(p->q_vecs[size_t(i) * DIM]) * 1000003LL;
    if (p->mode != OC_MODE_VECTOR) {
        for (uint32_t t = p->q_token_offsets[i]; t < p->q_token_offsets[i + 1]; t++)
            for (uint32_t e = p->token_term_offsets[t]; e < p->token_term_offsets[t + 1]; e++)
                sig += (long long)p->term_field[e] * 131 + (long long)p->term_id[e] * 7 +
                       (long long)llround((p->term_weight ? p->term_weight[e] : 1.0f) * 4) + 13LL * (t - p->q_token_offsets[i]);
    }
    return sig;
}
static uint64_t n_terms_of(const oc_search_params *p, uint32_t i) {
    if (p->mode == OC_MODE_VECTOR) return 0;
    const uint32_t t0 = p->q_token_offsets[i], t1 = p->q_token_offsets[i + 1];
    return (uint64_t)(p->token_term_offsets[t1] - p->token_term_offsets[t0]) + 1000ull * (t1 - t0);
}
static float score_of(int filter, uint32_t j, float similarity) { return float(filter * 1000) + 0.5f * j + similarity; }
// a query's filter as the executor sees it: q_filters[i], else the call's filter / host bitmap
static int filter_of(const oc_search_params *p, uint32_t i) {
    if (p->q_filters) return p->q_filters[i] ? index_of(p->q_filters[i], g_handles, N_HANDLES) : -1;
    if (p->filter) return index_of(p->filter, g_handles, N_HANDLES);
    return p->filter_bits ? 100 : -1;
}
static long long id_of(const oc_search_params *p, uint32_t i) {   // -1: a fulltext call carries no vector
    return p->mode == OC_MODE_FULLTEXT ? -1 : llround(p->q_vecs[size_t(i) * DIM + DIM - 1]);
}
static bool flat(Kind k) { return k == ocb::PLAIN || k == ocb::SORTED; }

struct Seen {
    std::atomic<int> bad{0}, calls[4]{}, merged[4]{}, max_b[4]{}, oom{0}, mixed{0}, checked{0};
    std::atomic<int> q_filtered{0}, unfiltered{0}, bits{0}, dev_filter{0};
};
static Seen g;
static void note_max(std::atomic<int> &m, int v) {
    int prev = m.load();
    while (v > prev && !m.compare_exchange_weak(prev, v)) {}
}

struct Fake {
    int operator()(const ocb::Call &c) const {
        const oc_search_params *p = c.p;
        const uint32_t B = p->n_queries, L = p->limit;
        const uint64_t page = uint64_t(L) + p->offset;
        if (page > OC_MAX_TOPK) return OC_ERR_UNSUPPORTED;
        for (uint32_t i = 0; i < B; i++) {
            const uint32_t k = c.pins ? c.pins->q_pin_offsets[i + 1] - c.pins->q_pin_offsets[i] : 0;
            if (k > OC_MAX_TOPK || (k && c.pins->apply && 2 * page > OC_MAX_TOPK)) return OC_ERR_UNSUPPORTED;
            if (c.q_groups && c.q_groups[i].max_results > OC_MAX_TOPK) return OC_ERR_UNSUPPORTED;
        }
        if (c.q_groups && B > g_oom_above) { g.oom++; return OC_ERR_OOM; }
        g.calls[c.kind]++;
        if (B > 1) g.merged[c.kind]++;
        note_max(g.max_b[c.kind], (int)B);
        std::this_thread::sleep_for(std::chrono::microseconds(300));   // "device time": lets the next group fill up
        if (B > 1 && p->filter) g.bad++;   // device filters reach a merged call in q_filters only
        if (p->filter) g.dev_filter++;
        if (p->filter_bits) {
            if (B != 1 || p->q_filters) g.bad++;
            g.bits++;
        }
        if (p->q_filters) {
            bool any = false;
            for (uint32_t i = 0; i < B; i++) any = any || p->q_filters[i];
            if (!any) g.bad++;   // q_filters set although no query of the call is filtered
            g.q_filtered++;
        } else if (!p->filter && !p->filter_bits) {
            g.unfiltered++;
        }
        bool sort_or_item = false, has_plain = false;
        uint64_t row = 0;
        for (uint32_t i = 0; i < B; i++) {
            const long long sig = signature(p, i);
            const int f = filter_of(p, i);
            for (uint32_t j = 0; j < L; j++) {
                c.docs[size_t(i) * L + j] = uint64_t(sig * 1000 + j);
                c.scores[size_t(i) * L + j] = score_of(f, j, p->similarity);
            }
            if (L) c.n[i] = L;
            const uint32_t k0 = c.pins ? c.pins->q_pin_offsets[i] : 0, k1 = c.pins ? c.pins->q_pin_offsets[i + 1] : 0;
            c.count[i] = n_terms_of(p, i) + 1000000ull * (k1 - k0);
            const oc_sort *s = c.kind == ocb::SORTED ? &c.q_sorts[i] : c.q_groups ? &c.q_groups[i].sort : nullptr;
            sort_or_item = sort_or_item || (s && s->field) || k1 > k0;
            const int sf = s && s->field ? index_of(s->field, g_fields, N_FIELDS) : -1;
            for (uint32_t j = 0; c.sort_values && j < L; j++) c.sort_values[size_t(i) * L + j] = sort_value(sf, s ? s->order : 0);
            const long long id = id_of(p, i);
            if (id < 0) continue;
            if (id >= MAX_IDS) { g.bad++; return OC_ERR_INVALID; }
            const Desc &d = g_desc[id];
            has_plain = has_plain || d.kind == ocb::PLAIN;
            bool ok = !d.refused && (flat(d.kind) ? flat(c.kind) : d.kind == c.kind) && f == d.filter && k1 - k0 == d.k;
            if (c.kind == ocb::PLAIN) ok = ok && d.field < 0 && !d.k;   // a call with a sort or an item runs as SORTED
            else if (d.kind != ocb::PLAIN) ok = ok && sf == d.field && (sf < 0 || s->order == d.order);
            for (uint32_t j = k0; j < k1; j++) {
                ok = ok && c.pins->doc_ids[j] == uint64_t(id) * 10 + (j - k0) && (B == 1 || c.pins->apply);
                if (c.pin_scores) c.pin_scores[j] = float(id) + c.pins->positions[j] / 8.f;   // entry j of the CSR, as the library
                if (c.pin_present) c.pin_present[j] = uint8_t(j - k0 + 1);
            }
            if (c.q_groups) {
                const oc_group_req &q = c.q_groups[i];
                ok = ok && q.groups == (d.gb < 0 ? nullptr : gb(d.gb)) && q.max_results == d.m && c.group_stride >= need_of(d);
                for (uint64_t gi = 0; gi < n_groups_of(d); gi++, row++) {
                    c.g_n[row] = n_of(uint32_t(id), gi);
                    for (uint32_t j = 0; j < c.group_stride; j++) {
                        const bool in = j < c.g_n[row];
                        c.g_docs[row * c.group_stride + j] = in ? doc_of(uint32_t(id), gi, j) : 0;
                        c.g_scores[row * c.group_stride + j] = in ? float(j) : 0.f;
                        c.g_values[row * c.group_stride + j] = in ? double(id) + 0.5 : 0.0;
                    }
                }
            }
            if (c.kind == ocb::FACETED) {
                const uint32_t f0 = c.q_facet_offsets[i], f1 = c.q_facet_offsets[i + 1];
                ok = ok && c.facets == store(d.store) && f1 - f0 == d.nf;
                for (uint32_t j = f0; j < f1; j++) {
                    ok = ok && c.facet_reqs[j].field == facet_field(uint32_t(id), j - f0) && c.facet_reqs[j].variant == id;
                    c.f_counts[j] = facet_count(uint32_t(id), j - f0);
                }
            }
            if (!ok) g.bad++;
        }
        if (c.kind == ocb::SORTED && B > 1 && !sort_or_item) g.bad++;   // such a batch runs as PLAIN
        if (c.kind == ocb::SORTED && has_plain) g.mixed++;
        return 0;
    }
    int check(const oc_facets *, const oc_facet_req *reqs, uint32_t n) const {
        g.checked++;
        for (uint32_t j = 0; j < n; j++)
            if (reqs[j].field == BAD_FIELD) return OC_ERR_INVALID;
        return OC_OK;
    }
};
using Batcher = ocb::Batcher<Fake>;

// A vector query of limit L carrying its id.
struct Query {
    oc_search_params p{};
    float qv[DIM] = {};
    Query(uint32_t id, uint32_t L) {
        p.mode = OC_MODE_VECTOR; p.n_queries = 1; p.limit = L;
        p.threshold = -1.0f; p.bm25_k = 1.2f; p.bm25_b = 0.75f;
        qv[0] = qv[DIM - 1] = float(id); p.q_vecs = qv;
    }
};
// The hits the fake gives query p with k items.
static bool hits_ok(const oc_search_params *p, const uint64_t *docs, const float *scores, uint32_t n, uint64_t count, int filter,
                    uint32_t k) {
    const long long sig = signature(p, 0);
    bool ok = n == p->limit && count == n_terms_of(p, 0) + 1000000ull * k;
    for (uint32_t j = 0; ok && j < p->limit; j++)
        ok = docs[j] == uint64_t(sig * 1000 + j) && scores[j] == score_of(filter, j, p->similarity);
    return ok;
}
// The group rows the fake gives request id, at its own stride.
static bool rows_ok(uint32_t id, const uint64_t *gd, const float *gs, const double *gv, const uint32_t *gn) {
    const Desc &d = g_desc[id];
    bool ok = true;
    for (uint64_t gi = 0; gi < n_groups_of(d); gi++) {
        const uint32_t want = n_of(id, gi);
        ok = ok && gn[gi] == want;
        for (uint32_t j = 0; j < d.stride; j++) {
            const bool in = j < want;
            const size_t o = gi * d.stride + j;
            ok = ok && gd[o] == (in ? doc_of(id, gi, j) : 0) && gs[o] == (in ? float(j) : 0.f) && gv[o] == (in ? double(id) + 0.5 : 0.0);
        }
    }
    return ok;
}
static void run_threads(int T, const std::function<void(int)> &fn) {
    std::vector<std::thread> th;
    for (int t = 0; t < T; t++) th.emplace_back(fn, t);
    for (auto &x : th) x.join();
}
struct Stats { uint64_t q = 0, nb = 0, direct = 0; };
static Stats stats_of(Batcher &b) {
    Stats s;
    b.stats(&s.q, &s.nb, &s.direct);
    printf("queries=%llu batches=%llu direct=%llu calls=%d/%d/%d/%d merged=%d/%d/%d/%d max_batch=%d/%d/%d/%d oom=%d mixed=%d "
           "checked=%d q_filtered=%d unfiltered=%d bits=%d\n",
           (unsigned long long)s.q, (unsigned long long)s.nb, (unsigned long long)s.direct, g.calls[0].load(), g.calls[1].load(),
           g.calls[2].load(), g.calls[3].load(), g.merged[0].load(), g.merged[1].load(), g.merged[2].load(), g.merged[3].load(),
           g.max_b[0].load(), g.max_b[1].load(), g.max_b[2].load(), g.max_b[3].load(), g.oom.load(), g.mixed.load(),
           g.checked.load(), g.q_filtered.load(), g.unfiltered.load(), g.bits.load());
    return s;
}

// Plain requests of every mode, limit and similarity, with token CSRs at non-zero offsets and NULL weights; some with a
// host bitmap (not batchable: direct).
static int plain() {
    Batcher b(Fake{}, DIM, 32, 2000);
    std::atomic<int> wrong{0};
    const int T = 16, Q = 250;
    run_threads(T, [&](int t) {
        std::mt19937 rng(1234 + t);
        for (int it = 0; it < Q; it++) {
            const uint32_t id = uint32_t(t * Q + it);
            Query q(id, (rng() % 2) ? 10 : 5);
            oc_search_params &p = q.p;
            p.mode = (int)(rng() % 3);
            p.similarity = (rng() % 2) ? 0.0f : 0.7f;
            for (uint32_t d = 0; d + 1 < DIM; d++) q.qv[d] = (float)(rng() % 1000);
            const uint32_t base = rng() % 3;                 // non-zero-based token offsets must be honoured
            const uint32_t ntok = rng() % 5;
            std::vector<uint32_t> qto = {base, base + ntok}, tto(base + ntok + 1, 0), tf, ti;
            std::vector<float> tw;
            for (uint32_t k = 0; k < ntok; k++) {
                const uint32_t nt = rng() % 4;                // 0 terms = unknown token
                for (uint32_t e = 0; e < nt; e++) { tf.push_back(rng() % 3); ti.push_back(rng() % 5000); tw.push_back((float)(1 + rng() % 3)); }
                tto[base + k + 1] = (uint32_t)ti.size();
            }
            static const uint32_t z = 0;
            p.q_token_offsets = qto.data(); p.token_term_offsets = tto.data();
            p.term_field = tf.empty() ? &z : tf.data(); p.term_id = ti.empty() ? &z : ti.data();
            const bool null_w = rng() % 4 == 0;
            if (null_w) for (auto &w : tw) w = 1.0f;
            p.term_weight = (null_w || tw.empty()) ? nullptr : tw.data();
            uint64_t bits = ~0ull;
            Desc &d = g_desc[id];
            if (rng() % 10 == 0) { p.filter_bits = &bits; p.filter_nbits = 64; d.filter = 100; }
            std::vector<uint64_t> docs(p.limit); std::vector<float> sc(p.limit);
            uint32_t n = 0; uint64_t cnt = 0;
            ocb::Request r{{ocb::PLAIN, &p, docs.data(), sc.data(), &n, &cnt}};
            const char *why = nullptr;
            const int rc = b.submit(r, &why);
            if (rc != 0 || !hits_ok(&p, docs.data(), sc.data(), n, cnt, d.filter, 0)) wrong++;
        }
    });
    const Stats s = stats_of(b);
    printf("wrong=%d bad=%d\n", wrong.load(), g.bad.load());
    if (wrong.load() || g.bad.load()) return 1;
    if (s.q + s.direct != (uint64_t)T * Q) return 2;
    if (s.nb * 2 > s.q) return 3;          // coalescing must happen: on average >= 2 queries per batch
    if (g.max_b[ocb::PLAIN].load() > 32) return 4;
    return 0;
}

// Plain requests with a device filter of their own, none, or a host bitmap (direct); threads t % 3 == 0 never filter.
static int qfilters() {
    Batcher b(Fake{}, DIM, 32, 2000);
    std::atomic<int> wrong{0};
    const int T = 12, Q = 200;
    run_threads(T, [&](int t) {
        std::mt19937 rng(777 + t);
        for (int it = 0; it < Q; it++) {
            const uint32_t id = uint32_t(t * Q + it);
            Query q(id, 1);
            Desc &d = g_desc[id];
            const uint32_t kind = rng() % 10;
            uint64_t bits = ~0ull;
            if (t % 3 == 0) {
                // this thread never filters: batches made only of such requests must have q_filters == NULL
            } else if (kind < 6) {
                d.filter = (int)(rng() % N_HANDLES);
                q.p.filter = handle(d.filter);
            } else if (kind == 6) {
                q.p.filter_bits = &bits; q.p.filter_nbits = 64;   // host bitmap: direct
                d.filter = 100;
            }
            uint64_t doc = 0; float sc = 0.f; uint32_t n = 0; uint64_t cnt = 0;
            ocb::Request r{{ocb::PLAIN, &q.p, &doc, &sc, &n, &cnt}};
            const char *why = nullptr;
            const int rc = b.submit(r, &why);
            if (rc != 0 || !hits_ok(&q.p, &doc, &sc, n, cnt, d.filter, 0)) wrong++;
        }
    });
    const Stats s = stats_of(b);
    printf("wrong=%d bad=%d\n", wrong.load(), g.bad.load());
    if (wrong.load() || g.bad.load() || g.dev_filter.load()) return 1;   // device filters reach the executor in q_filters only
    if (s.q + s.direct != (uint64_t)T * Q) return 2;
    if (s.direct != (uint64_t)g.bits.load()) return 3;   // only host-bitmap requests bypass the queue
    if (s.nb * 2 > s.q) return 4;                        // coalescing happened
    if (g.q_filtered.load() == 0) return 5;              // filtered requests were batched
    if (g.unfiltered.load() == 0) return 6;              // and batches without any filter kept q_filters NULL
    return 0;
}

// One plain request and one sorted request whose items the library refuses for their size, with the same batch key: the
// second must run alone and get OC_ERR_UNSUPPORTED, the first must succeed (a batch of one after max_wait_us) instead
// of failing with it.
static int oversized_items_run_alone() {
    Batcher b(Fake{}, DIM, 2, 300000);
    struct Case { uint32_t limit, items; };
    const Case cases[] = {{600, 1}, {10, OC_MAX_TOPK + 1}};   // 2 x (limit + offset) > OC_MAX_TOPK; too many items
    for (const Case &cs : cases) {
        const uint32_t L = cs.limit, K = cs.items;
        g_desc[0] = Desc{};
        g_desc[1] = Desc{}; g_desc[1].kind = ocb::SORTED; g_desc[1].k = K;
        std::vector<uint64_t> docA(L, 7), docB(L, 7), pdoc(K);
        std::vector<float> scA(L), scB(L), ps(K, -1.f);
        std::vector<double> svB(L, -7.0);
        std::vector<uint32_t> ppos(K, 0);
        std::vector<uint8_t> pp(K, 0xee);
        for (uint32_t j = 0; j < K; j++) pdoc[j] = 10 + j;
        uint32_t off[2] = {0, K}, nA = 0, nB = 7;
        uint64_t cA = 0, cB = 7;
        oc_pins pins{off, pdoc.data(), ppos.data(), 1};
        int rcA = 1, rcB = 1;
        Query qa(0, L), qb(1, L);
        std::thread ta([&] {
            ocb::Request r{{ocb::PLAIN, &qa.p, docA.data(), scA.data(), &nA, &cA}};
            const char *why = nullptr;
            rcA = b.submit(r, &why);
        });
        std::thread tb([&] {
            std::this_thread::sleep_for(std::chrono::milliseconds(20));   // while the plain request waits for company
            ocb::Request r{{ocb::SORTED, &qb.p, docB.data(), scB.data(), &nB, &cB, svB.data(), ps.data(), pp.data(), &pins,
                            ocb::score_order()}};
            const char *why = nullptr;
            rcB = b.submit(r, &why);
        });
        ta.join(); tb.join();
        if (rcA != 0 || nA != L || docA[0] != 0) return 10;
        if (rcB != OC_ERR_UNSUPPORTED || nB != 7 || cB != 7 || docB[0] != 7 || svB[0] != -7.0 || ps[0] != -1.f) return 11;
    }
    Stats s;
    b.stats(&s.q, &s.nb, &s.direct);
    if (s.direct != 2 || s.q != 2 || s.nb != 2 || g.bad.load()) return 12;
    return 0;
}

// Plain requests (threads t % 4 == 0, some with a device filter) and sorted requests: a sort or score order, 0-3 items
// at an offset inside the caller's arrays, some with a device filter, a host bitmap or apply = 0 (direct), some
// malformed (refused).  Threads t % 4 == 1 never sort and never pin, so their batches may stay PLAIN.
static int sorted() {
    if (const int rc = oversized_items_run_alone()) {
        printf("oversized items: failed with %d\n", rc);
        return rc;
    }
    Batcher b(Fake{}, DIM, 32, 2000);
    std::atomic<int> wrong{0}, refused{0}, expect_refused{0};
    const int T = 12, Q = 200;
    run_threads(T, [&](int t) {
        std::mt19937 rng(4242 + t);
        for (int it = 0; it < Q; it++) {
            const uint32_t id = uint32_t(t * Q + it);
            Query q(id, 1);
            Desc &d = g_desc[id] = Desc{};   // ids 0 and 1 described the oversized requests
            uint64_t bits = ~0ull;
            const uint32_t fk = rng() % 10;
            if (fk < 5) { d.filter = (int)(rng() % N_HANDLES); q.p.filter = handle(d.filter); }
            else if (fk == 5) { q.p.filter_bits = &bits; q.p.filter_nbits = 64; d.filter = 100; }   // host bitmap: direct
            uint64_t doc = 0; float sc = 0.f; uint32_t n = 0; uint64_t cnt = 0;
            const char *why = nullptr;
            if (t % 4 == 0) {
                ocb::Request r{{ocb::PLAIN, &q.p, &doc, &sc, &n, &cnt}};
                if (b.submit(r, &why) != 0 || !hits_ok(&q.p, &doc, &sc, n, cnt, d.filter, 0)) wrong++;
                continue;
            }
            d.kind = ocb::SORTED;
            oc_sort srt{nullptr, OC_SORT_ASC};
            const bool with_sort = t % 4 != 1 && rng() % 3 != 0;
            if (with_sort) { d.field = (int)(rng() % N_FIELDS); d.order = (int)(rng() % 2); srt = oc_sort{field(d.field), d.order}; }
            d.k = t % 4 == 1 ? 0u : rng() % 4;
            uint32_t off[2] = {3, 3 + d.k};   // the items sit at an offset inside the caller's arrays
            uint64_t pdoc[8] = {};
            uint32_t ppos[8] = {};
            for (uint32_t j = 0; j < d.k; j++) { pdoc[3 + j] = uint64_t(id) * 10 + j; ppos[3 + j] = (uint32_t)(rng() % 20); }
            oc_pins pins{off, pdoc, ppos, 1};
            const bool with_pins = d.k > 0 || rng() % 2;
            const uint32_t bad = t % 4 == 1 ? 15u : rng() % 16;   // 0..2: a malformed request
            if (bad == 0) { srt = oc_sort{field(0), 7}; }                       // bad order
            else if (bad == 1) { off[1] = 1; }                                  // not monotone
            else if (bad == 2 && d.k) { pins.positions = nullptr; }             // NULL positions
            d.refused = bad == 0 || bad == 1 || (bad == 2 && d.k);
            const bool use_pins = with_pins || bad == 1 || (bad == 2 && d.k);
            if (!d.refused && d.k && rng() % 8 == 0) pins.apply = d.apply = 0;   // direct
            double sv = -7.0; float ps[8]; uint8_t pp[8];
            for (int j = 0; j < 8; j++) { ps[j] = -1.f; pp[j] = 0xee; }
            ocb::Request r{{ocb::SORTED, &q.p, &doc, &sc, &n, &cnt, &sv, ps, pp, use_pins ? &pins : nullptr,
                            (with_sort || bad == 0) ? &srt : ocb::score_order()}};
            const int rc = b.submit(r, &why);
            if (d.refused) {
                expect_refused++;
                if (rc == OC_ERR_INVALID && why && n == 0 && sv == -7.0 && ps[0] == -1.f) refused++;
                else wrong++;
                continue;
            }
            const double want_sv = sort_value(d.field, d.order);
            bool ok = rc == 0 && hits_ok(&q.p, &doc, &sc, n, cnt, d.filter, d.k);
            ok = ok && (std::isnan(want_sv) ? std::isnan(sv) : sv == want_sv);
            // item j is output entry off[0] + j, as in a call of its own; nothing is written around the items
            for (uint32_t j = 0; j < d.k; j++) ok = ok && ps[3 + j] == float(id) + ppos[3 + j] / 8.f && pp[3 + j] == j + 1;
            ok = ok && ps[2] == -1.f && pp[2] == 0xee && ps[3 + d.k] == -1.f && pp[3 + d.k] == 0xee;
            if (!ok) wrong++;
        }
    });
    const Stats s = stats_of(b);
    printf("refused=%d/%d wrong=%d bad=%d\n", refused.load(), expect_refused.load(), wrong.load(), g.bad.load());
    if (wrong.load() || g.bad.load()) return 1;
    if (refused.load() != expect_refused.load() || refused.load() == 0) return 2;
    if (s.q + s.direct + refused.load() != (uint64_t)T * Q) return 3;   // every valid request ran exactly once
    if (s.nb * 2 > s.q) return 4;                                       // coalescing happened
    if (g.merged[ocb::SORTED].load() == 0 || g.merged[ocb::PLAIN].load() == 0) return 5;   // both merged kinds ran
    if (g.mixed.load() == 0) return 6;                                  // plain and sorted requests shared batches
    if (g.calls[ocb::SORTED].load() == g.merged[ocb::SORTED].load()) return 7;   // host-bitmap / apply = 0 requests ran alone
    return 0;
}

// Plain requests and grouped requests: a groupBy handle of 1, 3 or 7 groups or none, max_results 0-10, a sort or score
// order, 0-2 items, a group stride of its need plus 0-3.  Some have a stride below their need (refused) or
// max_results > OC_MAX_TOPK (the merged call would refuse it: it runs alone).  A merged call of more than 5 requests
// runs out of device memory.
static int groups() {
    std::mt19937 rng(7);
    const int T = 12, Q = 150, N = T * Q;
    std::vector<bool> oversized(N);
    for (int id = 0; id < N; id++) {
        Desc &d = g_desc[id];
        const int kind = int(rng() % 20);
        if (kind < 4) continue;
        d.kind = ocb::GROUPED;
        oversized[id] = kind == 5;
        d.gb = int(rng() % (N_GB + 1)) - 1;
        if (d.gb < 0 && kind == 5) d.gb = 0;
        d.m = oversized[id] ? OC_MAX_TOPK + 1 : uint32_t(rng() % 11);
        d.k = oversized[id] ? 0 : uint32_t(rng() % 3);
        d.field = int(rng() % (N_FIELDS + 1)) - 1;
        d.order = int(rng() % 2);
        d.stride = need_of(d) + uint32_t(rng() % 4);
        if (kind == 4) { d.refused = true; d.gb = 1; d.m = 4; d.stride = need_of(d) - 1; }
    }
    g_oom_above = 5;
    Batcher b(Fake{}, DIM, 32, 2000, true, false);
    std::atomic<int> wrong{0}, refused{0}, oversized_refused{0};
    const uint32_t L = 3;
    run_threads(T, [&](int t) {
        for (int id = t; id < N; id += T) {
            const Desc &d = g_desc[id];
            Query q(uint32_t(id), L);
            std::vector<uint64_t> docs(L, 7);
            std::vector<float> scores(L, 7.f);
            uint32_t n = 7;
            uint64_t count = 7;
            const char *why = nullptr;
            if (d.kind == ocb::PLAIN) {
                ocb::Request r{{ocb::PLAIN, &q.p, docs.data(), scores.data(), &n, &count}};
                if (b.submit(r, &why) != 0 || !hits_ok(&q.p, docs.data(), scores.data(), n, count, -1, 0)) wrong++;
                continue;
            }
            const oc_group_req req{d.gb < 0 ? nullptr : gb(d.gb), d.m, oc_sort{d.field < 0 ? nullptr : field(d.field), d.order}};
            std::vector<uint32_t> off = {0, d.k};
            std::vector<uint64_t> pdoc(std::max<uint32_t>(d.k, 1));
            std::vector<uint32_t> ppos(std::max<uint32_t>(d.k, 1), 0);
            for (uint32_t j = 0; j < d.k; j++) pdoc[j] = uint64_t(id) * 10 + j;
            const oc_pins pins{off.data(), pdoc.data(), ppos.data(), 1};
            const uint64_t G = n_groups_of(d);
            const size_t cells = std::max<size_t>(G * d.stride, 1);
            std::vector<uint64_t> gd(cells, 7);
            std::vector<float> gs(cells, 7.f);
            std::vector<double> gv(cells, 7.0), sv(L, 7.0);
            std::vector<uint32_t> gn(std::max<uint64_t>(G, 1), 7);
            std::vector<float> ps(2, 7.f);
            std::vector<uint8_t> pp(2, 7);
            ocb::Request r{{ocb::GROUPED, &q.p, docs.data(), scores.data(), &n, &count, sv.data(), ps.data(), pp.data(), &pins,
                            nullptr, &req, d.stride, gd.data(), gs.data(), gv.data(), gn.data()}, G};
            const int rc = b.submit(r, &why);
            if (d.refused) {
                if (rc != OC_ERR_INVALID || !why || gd[0] != 7 || gn[0] != 7 || n != 7) wrong++;
                refused++;
                continue;
            }
            if (oversized[id]) {
                if (rc != OC_ERR_UNSUPPORTED || n != 7) wrong++;
                oversized_refused++;
                continue;
            }
            const double want_sv = sort_value(d.field, d.order);
            bool ok = rc == 0 && hits_ok(&q.p, docs.data(), scores.data(), n, count, -1, d.k);
            ok = ok && (std::isnan(want_sv) ? std::isnan(sv[0]) : sv[0] == want_sv);
            if (!ok || !rows_ok(uint32_t(id), gd.data(), gs.data(), gv.data(), gn.data())) wrong++;
        }
    });
    const Stats s = stats_of(b);
    int bad = g.bad.load();
    if (g.merged[ocb::GROUPED].load() == 0 || refused.load() == 0 || oversized_refused.load() == 0) bad++;
    if (g.oom.load() == 0 || g.max_b[ocb::GROUPED].load() > (int)g_oom_above || s.nb >= s.q) bad++;
    printf("refused=%d oversized=%d wrong=%d bad=%d\n", refused.load(), oversized_refused.load(), wrong.load(), bad);
    return wrong.load() == 0 && bad == 0 ? 0 : 1;
}

// Plain, grouped and faceted requests: faceted ones on one of two stores, 0-4 facet requests, with or without a groupBy
// handle of 1 or 3 groups; some with a facet request the check refuses.  A merged call of more than 5 requests runs out
// of device memory.
static int facets() {
    std::mt19937 rng(11);
    const int T = 12, Q = 150, N = T * Q, MAX_F = 4;
    for (int id = 0; id < N; id++) {
        Desc &d = g_desc[id];
        const int k = int(rng() % 20);
        d.kind = k < 3 ? ocb::PLAIN : k < 6 ? ocb::GROUPED : ocb::FACETED;
        d.refused = k == 6;
        const int st = int(rng() % N_STORES);
        const int gbi = d.kind == ocb::GROUPED ? 0 : int(rng() % 3) - 1;
        const uint32_t nf = uint32_t(rng() % (MAX_F + 1));
        if (d.kind == ocb::PLAIN) continue;
        d.gb = gbi; d.m = d.gb < 0 ? 0 : 1; d.stride = 1;
        if (d.kind == ocb::FACETED) { d.store = st; d.nf = d.refused && nf == 0 ? 1 : nf; }
    }
    g_oom_above = 5;
    Batcher b(Fake{}, DIM, 32, 2000, true, false);
    std::atomic<int> wrong{0}, refused{0};
    const uint32_t L = 3;
    run_threads(T, [&](int t) {
        for (int id = t; id < N; id += T) {
            const Desc &d = g_desc[id];
            Query q(uint32_t(id), L);
            std::vector<uint64_t> docs(L, 7), gd(8, 7), fc(MAX_F + 1, 7);
            std::vector<float> scores(L, 7.f), gs(8, 7.f);
            std::vector<double> sv(L, 7.0), gv(8, 7.0);
            std::vector<uint32_t> gn(4, 7);
            uint32_t n = 7;
            uint64_t count = 7;
            const char *why = nullptr;
            if (d.kind == ocb::PLAIN) {
                ocb::Request r{{ocb::PLAIN, &q.p, docs.data(), scores.data(), &n, &count}};
                if (b.submit(r, &why) != 0 || !hits_ok(&q.p, docs.data(), scores.data(), n, count, -1, 0)) wrong++;
                continue;
            }
            const oc_group_req req{d.gb < 0 ? nullptr : gb(d.gb), d.m, oc_sort{nullptr, OC_SORT_ASC}};
            std::vector<oc_facet_req> fr(std::max<uint32_t>(d.nf, 1));
            for (uint32_t j = 0; j < d.nf; j++) fr[j] = oc_facet_req{facet_field(uint32_t(id), j), uint32_t(id), 0.0, 0.0};
            ocb::Request r{{d.kind, &q.p, docs.data(), scores.data(), &n, &count, sv.data(), nullptr, nullptr, nullptr, nullptr,
                            d.gb < 0 ? ocb::no_groups() : &req, 1, gd.data(), gs.data(), gv.data(), gn.data()},
                           n_groups_of(d), {0, d.nf}};
            if (d.kind == ocb::FACETED) {
                r.call.facets = store(d.store); r.call.q_facet_offsets = r.f_off; r.call.facet_reqs = fr.data();
                r.call.f_counts = fc.data();
            }
            const int rc = b.submit(r, &why);
            if (d.refused) {
                if (rc != OC_ERR_INVALID || n != 7 || count != 7 || fc[0] != 7) wrong++;
                refused++;
                continue;
            }
            bool ok = rc == 0 && hits_ok(&q.p, docs.data(), scores.data(), n, count, -1, 0) &&
                      rows_ok(uint32_t(id), gd.data(), gs.data(), gv.data(), gn.data());
            for (uint32_t j = 0; j < d.nf; j++) ok = ok && fc[j] == facet_count(uint32_t(id), j);
            ok = ok && fc[d.nf] == 7;   // nothing past its own counts
            if (!ok) wrong++;
        }
    });
    const Stats s = stats_of(b);
    int bad = g.bad.load();
    if (g.merged[ocb::FACETED].load() == 0 || refused.load() == 0 || s.direct != 0) bad++;
    if (g.oom.load() == 0 || g.max_b[ocb::FACETED].load() > (int)g_oom_above || s.nb >= s.q) bad++;
    printf("refused=%d wrong=%d bad=%d\n", refused.load(), wrong.load(), bad);
    return wrong.load() == 0 && bad == 0 ? 0 : 1;
}

int main(int argc, char **argv) {
    const struct { const char *name; int (*fn)(); } scenarios[] = {
        {"plain", plain}, {"qfilters", qfilters}, {"sorted", sorted}, {"groups", groups}, {"facets", facets}};
    for (const auto &s : scenarios)
        if (argc == 2 && strcmp(argv[1], s.name) == 0) return s.fn();
    fprintf(stderr, "usage: %s plain | qfilters | sorted | groups | facets\n", argv[0]);
    return 100;
}
