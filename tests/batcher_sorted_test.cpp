// Host-logic test of sorted and pinned requests in the micro-batching queue (oramacore_b200/csrc/batcher.h) with fake
// executors: 12 threads submit single queries through submit() (plain, some with a device filter) and submit_sorted()
// (a sort or score order, 0-3 promote items, some with a device filter, some malformed).  It checks that
//   - a merged batch with a sort or an item reaches the sorted executor with each request's sort, items and filter at
//     its own position (q_sorts[b], the items CSR, q_filters[b]), and a batch with neither reaches the plain executor;
//   - sort values and per-item pin outputs go back to the caller they belong to;
//   - malformed requests are refused with OC_ERR_INVALID and never reach an executor;
//   - host-bitmap and apply = 0 requests run directly, alone;
//   - a request whose items the library refuses for their size runs alone and gets that refusal, while a plain request
//     that would have shared its batch succeeds.
// Built and run by tests/test_batcher_sorted_host.py (g++, no CUDA).
#include <atomic>
#include <cmath>
#include <cstdio>
#include <random>
#include <thread>
#include <vector>

#include "../oramacore_b200/csrc/batcher.h"

static const uint32_t DIM = 4;
static const int N_HANDLES = 5, N_FIELDS = 3;
static char g_handles[N_HANDLES], g_fields[N_FIELDS];   // fake handles: only their addresses are used
static const oc_filter *handle(int i) { return reinterpret_cast<const oc_filter *>(&g_handles[i]); }
static const oc_sort_field *field(int i) { return reinterpret_cast<const oc_sort_field *>(&g_fields[i]); }
static int handle_index(const oc_filter *f) {
    for (int i = 0; i < N_HANDLES; i++) if (f == handle(i)) return i;
    return -2;
}
static int field_index(const oc_sort_field *f) {
    for (int i = 0; i < N_FIELDS; i++) if (f == field(i)) return i;
    return -2;
}
static const int T = 12, Q = 200, N_IDS = T * Q;
static std::atomic<int> g_invalid[N_IDS];   // 1: a request that must be refused before it reaches an executor
static std::atomic<int> g_plain[N_IDS];     // 1: a request of submit()

struct Seen {
    std::atomic<int> bad{0}, plain_batches{0}, sorted_batches{0}, mixed_batches{0}, direct{0}, max_batch{0};
};
static void note_batch(Seen *s, uint32_t B) {
    int prev = s->max_batch.load();
    while ((int)B > prev && !s->max_batch.compare_exchange_weak(prev, (int)B)) {}
}
// a query's filter as the executor sees it: q_filters[i], else the batch-wide filter / host bitmap (-1 = none)
static int filter_of(const oc_search_params *p, uint32_t i) {
    if (p->q_filters) return p->q_filters[i] ? handle_index(p->q_filters[i]) : -1;
    if (p->filter) return handle_index(p->filter);
    return p->filter_bits ? 100 : -1;
}
static uint32_t id_of(const oc_search_params *p, uint32_t i) { return (uint32_t)llround(p->q_vecs[size_t(i) * DIM]); }

// The plain search: docs = the query's id, scores = its filter, count = 0 (no item).  It refuses what oc_search refuses
// for the page size.
struct FakeExec {
    Seen *s;
    int operator()(const oc_search_params *p, uint64_t *docs, float *scores, uint32_t *n, uint64_t *count) const {
        if (uint64_t(p->limit) + p->offset > OC_MAX_TOPK) return OC_ERR_UNSUPPORTED;
        note_batch(s, p->n_queries);
        std::this_thread::sleep_for(std::chrono::microseconds(200));
        if (p->n_queries > 1 && p->filter) s->bad++;   // device filters reach a merged executor in q_filters only
        if (p->n_queries > 1) s->plain_batches++;
        for (uint32_t i = 0; i < p->n_queries; i++) {
            const uint32_t id = id_of(p, i);
            if (id >= (uint32_t)N_IDS || g_invalid[id]) { s->bad++; continue; }
            docs[size_t(i) * p->limit] = id; scores[size_t(i) * p->limit] = (float)filter_of(p, i); n[i] = 1; count[i] = 0;
        }
        return 0;
    }
};
// The sorted search: as FakeExec, plus sort value = 2 * field + order (NaN in score order), count = the query's items,
// and per item: score = id + position / 8, present = its index inside the query + 1.  It refuses what
// oc_search_q_sorted refuses for the sizes: the page, a query with more than OC_MAX_TOPK items, and any query with items
// when 2 x (limit + offset) > OC_MAX_TOPK.
struct FakeSortedExec {
    Seen *s;
    int operator()(const oc_search_params *p, const oc_sort *q_sorts, const oc_pins *pins, uint64_t *docs, float *scores,
                   double *sort_values, uint32_t *n, uint64_t *count, float *pin_scores, uint8_t *pin_present) const {
        const uint64_t page = uint64_t(p->limit) + p->offset;
        if (page > OC_MAX_TOPK) return OC_ERR_UNSUPPORTED;
        for (uint32_t i = 0; pins && i < p->n_queries; i++) {
            const uint32_t k = pins->q_pin_offsets[i + 1] - pins->q_pin_offsets[i];
            if (k > OC_MAX_TOPK || (pins->apply && k && 2 * page > OC_MAX_TOPK)) return OC_ERR_UNSUPPORTED;
        }
        note_batch(s, p->n_queries);
        std::this_thread::sleep_for(std::chrono::microseconds(200));
        if ((p->n_queries > 1 && p->filter) || !q_sorts || !sort_values) s->bad++;
        if (p->n_queries > 1) s->sorted_batches++;
        else s->direct++;
        bool any = false, mixed = false;
        for (uint32_t i = 0; i < p->n_queries; i++) {
            const uint32_t id = id_of(p, i);
            if (id >= (uint32_t)N_IDS || g_invalid[id]) { s->bad++; continue; }
            mixed = mixed || g_plain[id];
            docs[size_t(i) * p->limit] = id; scores[size_t(i) * p->limit] = (float)filter_of(p, i); n[i] = 1;
            const oc_sort &st = q_sorts[i];
            if (st.field) { any = true; if (field_index(st.field) < 0) s->bad++; }
            sort_values[size_t(i) * p->limit] = st.field ? double(2 * field_index(st.field) + st.order) : std::nan("");
            const uint32_t k0 = pins ? pins->q_pin_offsets[i] : 0, k1 = pins ? pins->q_pin_offsets[i + 1] : 0;
            any = any || k1 > k0;
            count[i] = k1 - k0;
            for (uint32_t j = k0; j < k1; j++) {
                if (pins->doc_ids[j] != uint64_t(id) * 10 + (j - k0) || (p->n_queries > 1 && !pins->apply)) s->bad++;
                if (pin_scores) pin_scores[j] = float(id) + pins->positions[j] / 8.f;   // entry j of the CSR, as the library
                if (pin_present) pin_present[j] = uint8_t(j - k0 + 1);
            }
        }
        if (p->n_queries > 1 && !any) s->bad++;   // a merged batch with no sort and no item belongs to FakeExec
        if (mixed) s->mixed_batches++;
        return 0;
    }
};

// One plain request through submit() and one through submit_sorted() whose items the library refuses for their size,
// submitted together with the same batch key: the second must run alone and get OC_ERR_UNSUPPORTED, the first must
// succeed (a batch of one after max_wait_us) instead of failing with it.
static int oversized_items_run_alone() {
    Seen seen;
    ocb::Batcher<FakeExec, FakeSortedExec> b(FakeExec{&seen}, DIM, 2, 300000, true, true, FakeSortedExec{&seen});
    struct Case { uint32_t limit, items; };
    const Case cases[] = {{600, 1}, {10, OC_MAX_TOPK + 1}};   // 2 x (limit + offset) > OC_MAX_TOPK; too many items
    for (const Case &cs : cases) {
        const uint32_t L = cs.limit, K = cs.items;
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
        auto params = [&](oc_search_params &p, float *qv) {
            p.mode = OC_MODE_VECTOR; p.n_queries = 1; p.limit = L;
            p.threshold = -1.0f; p.bm25_k = 1.2f; p.bm25_b = 0.75f; p.q_vecs = qv;
        };
        std::thread ta([&] {
            oc_search_params p{}; float qv[DIM] = {0.f, 0.f, 0.f, 0.f}; params(p, qv);
            rcA = b.submit(&p, docA.data(), scA.data(), &nA, &cA);
        });
        std::thread tb([&] {
            std::this_thread::sleep_for(std::chrono::milliseconds(20));   // while the plain request waits for company
            oc_search_params p{}; float qv[DIM] = {1.f, 0.f, 0.f, 0.f}; params(p, qv);
            rcB = b.submit_sorted(&p, nullptr, &pins, docB.data(), scB.data(), svB.data(), &nB, &cB, ps.data(), pp.data());
        });
        ta.join(); tb.join();
        if (rcA != 0 || nA != 1 || docA[0] != 0) return 10;
        if (rcB != OC_ERR_UNSUPPORTED || nB != 7 || cB != 7 || docB[0] != 7 || svB[0] != -7.0 || ps[0] != -1.f) return 11;
    }
    uint64_t q = 0, nb = 0, direct = 0;
    b.stats(&q, &nb, &direct);
    if (direct != 2 || q != 2 || nb != 2 || seen.bad.load()) return 12;
    return 0;
}

int main() {
    if (const int rc = oversized_items_run_alone()) {
        printf("oversized items: failed with %d\n", rc);
        return rc;
    }
    Seen seen;
    ocb::Batcher<FakeExec, FakeSortedExec> b(FakeExec{&seen}, DIM, 32, 2000, true, true, FakeSortedExec{&seen});
    std::atomic<int> wrong{0}, refused{0}, expect_refused{0};
    std::vector<std::thread> th;
    for (int t = 0; t < T; t++)
        th.emplace_back([&, t] {
            std::mt19937 rng(4242 + t);
            for (int it = 0; it < Q; it++) {
                const uint32_t id = uint32_t(t * Q + it);
                oc_search_params p{};
                p.mode = OC_MODE_VECTOR;
                p.n_queries = 1;
                p.limit = 1;
                p.threshold = -1.0f; p.bm25_k = 1.2f; p.bm25_b = 0.75f;
                float qv[DIM] = {(float)id, 0.f, 0.f, 0.f};
                p.q_vecs = qv;
                int expect_f = -1;
                uint64_t bits = ~0ull;
                const uint32_t fk = rng() % 10;
                if (fk < 5) { expect_f = (int)(rng() % N_HANDLES); p.filter = handle(expect_f); }
                else if (fk == 5) { p.filter_bits = &bits; p.filter_nbits = 64; expect_f = 100; }   // host bitmap: direct
                uint64_t doc = 0; float sc = 0.f; uint32_t n = 0; uint64_t cnt = 0;
                if (t % 4 == 0) {   // plain requests through submit()
                    g_plain[id] = 1;
                    const int rc = b.submit(&p, &doc, &sc, &n, &cnt);
                    if (rc != 0 || n != 1 || doc != id || sc != (float)expect_f || cnt != 0) wrong++;
                    continue;
                }
                // sorted / pinned requests: t % 4 == 1 never sorts and never pins (their batches may stay plain)
                oc_sort srt{nullptr, OC_SORT_ASC};
                const bool sorted = t % 4 != 1 && rng() % 3 != 0;
                if (sorted) srt = oc_sort{field((int)(rng() % N_FIELDS)), (int)(rng() % 2)};
                const uint32_t k = t % 4 == 1 ? 0u : rng() % 4;
                uint32_t off[2] = {3, 3 + k};   // the items sit at an offset inside the caller's arrays
                uint64_t pdoc[8] = {};
                uint32_t ppos[8] = {};
                for (uint32_t j = 0; j < k; j++) { pdoc[3 + j] = uint64_t(id) * 10 + j; ppos[3 + j] = (uint32_t)(rng() % 20); }
                oc_pins pins{off, pdoc, ppos, 1};
                const bool with_pins = k > 0 || rng() % 2;
                const uint32_t bad = t % 4 == 1 ? 15u : rng() % 16;   // 0..2: a malformed request
                if (bad == 0) { srt = oc_sort{field(0), 7}; }                       // bad order
                else if (bad == 1) { off[1] = 1; }                                  // not monotone
                else if (bad == 2 && k) { pins.positions = nullptr; }               // NULL positions
                const bool invalid = bad == 0 || bad == 1 || (bad == 2 && k);
                const bool use_pins = with_pins || bad == 1 || (bad == 2 && k);
                const bool direct_apply0 = !invalid && k && rng() % 8 == 0;
                if (direct_apply0) pins.apply = 0;
                g_invalid[id] = invalid ? 1 : 0;
                double sv = -7.0; float ps[8]; uint8_t pp[8];
                for (int j = 0; j < 8; j++) { ps[j] = -1.f; pp[j] = 0xee; }
                const int rc = b.submit_sorted(&p, (sorted || bad == 0) ? &srt : nullptr, use_pins ? &pins : nullptr, &doc, &sc, &sv, &n,
                                               &cnt, ps, pp);
                if (invalid) {
                    expect_refused++;
                    if (rc == OC_ERR_INVALID && n == 0 && sv == -7.0 && ps[0] == -1.f) refused++;
                    else wrong++;
                    continue;
                }
                const double want_sv = sorted ? double(2 * field_index(srt.field) + srt.order) : std::nan("");
                bool ok = rc == 0 && n == 1 && doc == id && sc == (float)expect_f;
                ok = ok && (std::isnan(want_sv) ? std::isnan(sv) : sv == want_sv);
                ok = ok && cnt == k;
                // item j is output entry off[0] + j, as in a call of its own; nothing is written around the items
                for (uint32_t j = 0; j < k; j++) ok = ok && ps[3 + j] == float(id) + ppos[3 + j] / 8.f && pp[3 + j] == j + 1;
                ok = ok && ps[2] == -1.f && pp[2] == 0xee && ps[3 + k] == -1.f && pp[3 + k] == 0xee;
                if (!ok) wrong++;
            }
        });
    for (auto &x : th) x.join();
    uint64_t q = 0, nb = 0, direct = 0;
    b.stats(&q, &nb, &direct);
    const int bad = seen.bad.load();
    printf("queries=%llu batches=%llu direct=%llu plain_batches=%d sorted_batches=%d mixed_batches=%d max_batch=%d refused=%d/%d "
           "wrong=%d bad=%d\n",
           (unsigned long long)q, (unsigned long long)nb, (unsigned long long)direct, seen.plain_batches.load(),
           seen.sorted_batches.load(), seen.mixed_batches.load(), seen.max_batch.load(), refused.load(), expect_refused.load(),
           wrong.load(), bad);
    if (wrong.load() || bad) return 1;
    if (refused.load() != expect_refused.load() || refused.load() == 0) return 2;
    if (q + direct + refused.load() != (uint64_t)N_IDS) return 3;   // every valid request ran exactly once
    if (nb * 2 > q) return 4;                                       // coalescing happened
    if (seen.sorted_batches.load() == 0 || seen.plain_batches.load() == 0) return 5;   // both merged executors were used
    if (seen.mixed_batches.load() == 0) return 6;                   // plain and sorted requests shared batches
    if (seen.direct.load() == 0) return 7;                          // host-bitmap / apply = 0 requests ran alone
    return 0;
}
