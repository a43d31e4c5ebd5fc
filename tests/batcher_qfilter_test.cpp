// Host-logic test of per-query device filters in the micro-batching queue (oramacore_b200/csrc/batcher.h) with a fake
// executor: 12 threads submit single queries, some with their own device filter (p->filter), some without, some with a
// host bitmap (filter_bits).  A merged batch must carry each request's filter at its position in q_filters, NULL for an
// unfiltered request and a NULL q_filters array when no request of the batch is filtered; filter_bits requests must
// run directly.  Built and run by tests/test_batcher_qfilters_host.py (g++, no CUDA).
#include <atomic>
#include <cmath>
#include <cstdio>
#include <random>
#include <thread>
#include <vector>

#include "../oramacore_b200/csrc/batcher.h"

static const uint32_t DIM = 4;
static const int N_HANDLES = 7;
static char g_handles[N_HANDLES];   // fake oc_filter handles: only their addresses are used
static const oc_filter *handle(int i) { return reinterpret_cast<const oc_filter *>(&g_handles[i]); }
static int handle_index(const oc_filter *f) {
    for (int i = 0; i < N_HANDLES; i++) if (f == handle(i)) return i;
    return -2;
}

struct Seen { std::atomic<int> bad{0}, merged_filtered{0}, merged_plain{0}, direct_bits{0}, max_batch{0}; };

// The fake search: a query's answer encodes its id (q_vecs[0]) and the filter it was executed under
// (-1 = none).  Merged calls must come with q_filters (or NULL) and never with filter / filter_bits.
struct FakeExec {
    Seen *s;
    int operator()(const oc_search_params *p, uint64_t *docs, float *scores, uint32_t *n, uint64_t *count) const {
        int prev = s->max_batch.load();
        while ((int)p->n_queries > prev && !s->max_batch.compare_exchange_weak(prev, (int)p->n_queries)) {}
        std::this_thread::sleep_for(std::chrono::microseconds(200));
        if (p->filter) s->bad++;   // device filters are batchable: they reach the executor in q_filters only
        if (p->filter_bits) {
            if (p->n_queries != 1 || p->q_filters) s->bad++;
            s->direct_bits++;
        }
        bool any = false;
        for (uint32_t i = 0; i < p->n_queries; i++) {
            int f = -1;
            if (p->q_filters) {
                if (p->q_filters[i]) { f = handle_index(p->q_filters[i]); any = true; }
            } else if (p->filter) {
                f = handle_index(p->filter);
            } else if (p->filter_bits) {
                f = 100;
            }
            docs[i] = (uint64_t)llround(p->q_vecs[size_t(i) * DIM]);
            scores[i] = (float)f;
            n[i] = 1;
            count[i] = p->n_queries;
        }
        if (p->q_filters && !any) s->bad++;   // q_filters set although no request of the batch is filtered
        if (p->q_filters) s->merged_filtered++;
        else if (!p->filter_bits) s->merged_plain++;
        return 0;
    }
};

int main() {
    Seen seen;
    ocb::Batcher<FakeExec> b(FakeExec{&seen}, DIM, 32, 2000);
    std::atomic<int> wrong{0};
    const int T = 12, Q = 200;
    std::vector<std::thread> th;
    for (int t = 0; t < T; t++)
        th.emplace_back([&, t] {
            std::mt19937 rng(777 + t);
            for (int it = 0; it < Q; it++) {
                const int id = t * Q + it;
                oc_search_params p{};
                p.mode = OC_MODE_VECTOR;
                p.n_queries = 1;
                p.limit = 1;
                p.threshold = -1.0f; p.bm25_k = 1.2f; p.bm25_b = 0.75f;
                float qv[DIM] = {(float)id, 0.f, 0.f, 0.f};
                p.q_vecs = qv;
                int expect = -1;
                const uint32_t kind = rng() % 10;
                uint64_t bits = ~0ull;
                if (t % 3 == 0) {
                    // this thread never filters: batches made only of such requests must have q_filters == NULL
                } else if (kind < 6) {
                    expect = (int)(rng() % N_HANDLES);
                    p.filter = handle(expect);
                } else if (kind == 6) {
                    p.filter_bits = &bits; p.filter_nbits = 64;   // host bitmap: direct
                    expect = 100;
                }
                uint64_t doc = 0; float sc = 0.f; uint32_t n = 0; uint64_t cnt = 0;
                const int rc = b.submit(&p, &doc, &sc, &n, &cnt);
                if (rc != 0 || n != 1 || doc != (uint64_t)id || sc != (float)expect) wrong++;
            }
        });
    for (auto &x : th) x.join();
    uint64_t q = 0, nb = 0, direct = 0;
    b.stats(&q, &nb, &direct);
    printf("queries=%llu batches=%llu direct=%llu direct_bits=%d merged_filtered=%d merged_plain=%d max_batch=%d wrong=%d bad=%d\n",
           (unsigned long long)q, (unsigned long long)nb, (unsigned long long)direct, seen.direct_bits.load(),
           seen.merged_filtered.load(), seen.merged_plain.load(), seen.max_batch.load(), wrong.load(), seen.bad.load());
    if (wrong.load() || seen.bad.load()) return 1;
    if (q + direct != (uint64_t)T * Q) return 2;
    if (direct != (uint64_t)seen.direct_bits.load()) return 3;   // only host-bitmap requests bypass the queue
    if (nb * 2 > q) return 4;                                     // coalescing happened
    if (seen.merged_filtered.load() == 0) return 5;               // filtered requests were batched
    if (seen.merged_plain.load() == 0) return 6;                  // and batches without any filter kept q_filters NULL
    return 0;
}
