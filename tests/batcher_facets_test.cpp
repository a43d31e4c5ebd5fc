// Host-logic test of faceted requests in the micro-batching queue (oramacore_b200/csrc/batcher.h) with fake executors:
// 12 threads submit single queries through submit() (plain), submit_groups() (grouped) and submit_faceted() on one of
// two facet stores (0-4 facet requests, with or without a groupBy handle of 1 or 3 groups).  It checks that
//   - faceted requests never share a batch with plain or grouped requests, nor with requests on the other store, and
//     faceted requests do coalesce;
//   - the faceted executor sees each request's facet requests at its own range of q_facet_offsets, and each caller gets
//     back its own counts (and group rows);
//   - a merged call that fails with OC_ERR_OOM (here: any batch of more than 5 requests) is split in halves and every
//     request still succeeds;
//   - a request the executor's check refuses (an unknown field) gets OC_ERR_INVALID alone, never reaches an executor,
//     and the requests around it succeed.
// Built and run by tests/test_batcher_facets_host.py (g++, no CUDA).
#include <atomic>
#include <cmath>
#include <cstdio>
#include <random>
#include <thread>
#include <vector>

#include "../oramacore_b200/csrc/batcher.h"

static const uint32_t DIM = 4, LIMIT = 3, OOM_ABOVE = 5, BAD_FIELD = 99, MAX_F = 4;
static const int N_GB = 2, N_STORES = 2;
static const uint64_t GB_GROUPS[N_GB] = {1, 3};
static char g_gb[N_GB], g_st[N_STORES];   // fake handles: only their addresses are used
static const oc_group_by *gb(int i) { return reinterpret_cast<const oc_group_by *>(&g_gb[i]); }
static const oc_facets *store(int i) { return reinterpret_cast<const oc_facets *>(&g_st[i]); }
static const int T = 12, Q = 150, N_IDS = T * Q;

enum Kind { PLAIN, GROUPED, FACETED, REFUSED };
struct Req {
    Kind kind = PLAIN;
    int st = 0, gb = -1;                 // store; groupBy handle, -1: none
    uint32_t nf = 0;                     // facet requests
};
static Req g_req[N_IDS];
static uint32_t field_of(uint32_t id, uint32_t j) { return g_req[id].kind == REFUSED && j == 0 ? BAD_FIELD : (id + j) % 7; }
static uint64_t count_of(uint32_t id, uint32_t j) { return uint64_t(id) * 1000 + j + 1; }
static uint64_t doc_of(uint32_t id, uint64_t g) { return uint64_t(id) * 100 + g + 1; }

std::atomic<int> g_bad{0}, g_faceted_batches{0}, g_oom{0}, g_max_faceted{0}, g_checked{0};
static uint32_t id_of(const oc_search_params *p, uint32_t i) { return (uint32_t)llround(p->q_vecs[size_t(i) * DIM]); }

// every executor writes the flat outputs: docs[0] = id, n = 1, count = id
static void flat(const oc_search_params *p, uint32_t i, uint32_t id, uint64_t *docs, uint32_t *n, uint64_t *count) {
    docs[size_t(i) * p->limit] = id; n[i] = 1; count[i] = id;
}
struct FakeExec {
    int operator()(const oc_search_params *p, uint64_t *docs, float *, uint32_t *n, uint64_t *count) const {
        for (uint32_t i = 0; i < p->n_queries; i++) {
            const uint32_t id = id_of(p, i);
            if (id >= (uint32_t)N_IDS || g_req[id].kind != PLAIN) { g_bad++; continue; }
            flat(p, i, id, docs, n, count);
        }
        return 0;
    }
};
struct FakeGroupedExec {
    int operator()(const oc_search_params *p, const oc_group_req *, const oc_pins *, uint32_t, uint64_t *docs, float *, double *,
                   uint32_t *n, uint64_t *count, float *, uint8_t *, uint64_t *g_doc, float *, double *, uint32_t *g_n) const {
        uint64_t row = 0;
        for (uint32_t i = 0; i < p->n_queries; i++) {
            const uint32_t id = id_of(p, i);
            if (id >= (uint32_t)N_IDS || g_req[id].kind != GROUPED) { g_bad++; return OC_ERR_INVALID; }   // a faceted request here
            flat(p, i, id, docs, n, count);
            g_n[row] = 1; g_doc[row] = doc_of(id, 0); row++;
        }
        return 0;
    }
};
struct FakeFacetedExec {
    int operator()(const oc_search_params *p, const oc_group_req *q, const oc_pins *, uint32_t stride, const oc_facets *facets,
                   const uint32_t *off, const oc_facet_req *reqs, uint64_t *docs, float *, double *, uint32_t *n, uint64_t *count,
                   float *, uint8_t *, uint64_t *g_doc, float *, double *, uint32_t *g_n, uint64_t *f_counts) const {
        const uint32_t B = p->n_queries;
        if (B > OOM_ABOVE) { g_oom++; return OC_ERR_OOM; }
        if (B > 1) {
            g_faceted_batches++;
            int prev = g_max_faceted.load();
            while ((int)B > prev && !g_max_faceted.compare_exchange_weak(prev, (int)B)) {}
        }
        uint64_t row = 0;
        for (uint32_t i = 0; i < B; i++) {
            const uint32_t id = id_of(p, i);
            if (id >= (uint32_t)N_IDS) { g_bad++; return OC_ERR_INVALID; }
            const Req &r = g_req[id];
            // a plain, grouped or refused request, another store, or another request's facets
            if (r.kind != FACETED || facets != store(r.st) || off[i + 1] - off[i] != r.nf) g_bad++;
            if (r.gb < 0 ? q[i].groups != nullptr : q[i].groups != gb(r.gb)) g_bad++;
            flat(p, i, id, docs, n, count);
            for (uint32_t j = 0; j < off[i + 1] - off[i]; j++) {
                if (reqs[off[i] + j].field != field_of(id, j) || reqs[off[i] + j].variant != id) g_bad++;
                f_counts[off[i] + j] = count_of(id, j);
            }
            const uint64_t G = r.gb < 0 ? 0 : GB_GROUPS[r.gb];
            for (uint64_t g = 0; g < G; g++, row++) {
                g_n[row] = 1;
                for (uint32_t j = 0; j < stride; j++) g_doc[row * stride + j] = j == 0 ? doc_of(id, g) : 0;
            }
        }
        return 0;
    }
    int check(const oc_facets *, const oc_facet_req *reqs, uint32_t n) const {
        g_checked++;
        for (uint32_t j = 0; j < n; j++)
            if (reqs[j].field == BAD_FIELD) return OC_ERR_INVALID;
        return OC_OK;
    }
};

int main() {
    std::mt19937 rng(11);
    for (int id = 0; id < N_IDS; id++) {
        Req &r = g_req[id];
        const int k = int(rng() % 20);
        r.kind = k < 3 ? PLAIN : k < 6 ? GROUPED : k < 7 ? REFUSED : FACETED;
        r.st = int(rng() % N_STORES);
        r.gb = r.kind == GROUPED ? 0 : int(rng() % (N_GB + 1)) - 1;
        r.nf = uint32_t(rng() % (MAX_F + 1));
        if (r.kind == REFUSED && r.nf == 0) r.nf = 1;
    }
    ocb::Batcher<FakeExec, ocb::NoSortedExec, FakeGroupedExec, FakeFacetedExec> bat(FakeExec{}, DIM, 32, 2000, true, false);
    std::atomic<int> wrong{0}, refused{0};
    auto worker = [&](int t) {
        for (int id = t; id < N_IDS; id += T) {
            const Req &r = g_req[id];
            float qv[DIM] = {float(id), 0, 0, 0};
            oc_search_params p{};
            p.mode = OC_MODE_VECTOR; p.n_queries = 1; p.limit = LIMIT; p.q_vecs = qv;
            std::vector<uint64_t> docs(LIMIT, 7), gd(8, 7), fc(MAX_F + 1, 7);
            std::vector<float> scores(LIMIT, 7.f), gs(8, 7.f);
            std::vector<double> sv(LIMIT, 7.0), gv(8, 7.0);
            std::vector<uint32_t> gn(4, 7);
            uint32_t n = 7;
            uint64_t count = 7;
            if (r.kind == PLAIN) {
                const int rc = bat.submit(&p, docs.data(), scores.data(), &n, &count);
                if (rc != 0 || docs[0] != uint64_t(id) || n != 1 || count != uint64_t(id)) wrong++;
                continue;
            }
            const oc_group_req req{r.gb < 0 ? nullptr : gb(r.gb), 1, oc_sort{nullptr, OC_SORT_ASC}};
            const uint64_t G = r.gb < 0 ? 0 : GB_GROUPS[r.gb];
            if (r.kind == GROUPED) {
                const int rc = bat.submit_groups(&p, &req, G, nullptr, 1, docs.data(), scores.data(), sv.data(), &n, &count, nullptr,
                                                 nullptr, gd.data(), gs.data(), gv.data(), gn.data());
                if (rc != 0 || docs[0] != uint64_t(id) || gd[0] != doc_of(id, 0) || gn[0] != 1) wrong++;
                continue;
            }
            std::vector<oc_facet_req> fr(std::max<uint32_t>(r.nf, 1));
            for (uint32_t j = 0; j < r.nf; j++) fr[j] = oc_facet_req{field_of(id, j), uint32_t(id), 0.0, 0.0};
            const int rc = bat.submit_faceted(&p, store(r.st), fr.data(), r.nf, r.gb < 0 ? nullptr : &req, G, nullptr, 1, docs.data(),
                                              scores.data(), sv.data(), &n, &count, nullptr, nullptr, gd.data(), gs.data(), gv.data(),
                                              gn.data(), fc.data());
            if (r.kind == REFUSED) {
                if (rc != OC_ERR_INVALID || n != 7 || count != 7 || fc[0] != 7) wrong++;
                refused++;
                continue;
            }
            if (rc != 0 || docs[0] != uint64_t(id) || n != 1 || count != uint64_t(id)) { wrong++; continue; }
            for (uint32_t j = 0; j < r.nf; j++)
                if (fc[j] != count_of(id, j)) wrong++;
            if (fc[r.nf] != 7) wrong++;   // nothing past its own counts
            for (uint64_t g = 0; g < G; g++)
                if (gd[g] != doc_of(id, g) || gn[g] != 1) wrong++;
        }
    };
    std::vector<std::thread> th;
    for (int t = 0; t < T; t++) th.emplace_back(worker, t);
    for (auto &x : th) x.join();
    uint64_t queries = 0, batches = 0, direct = 0;
    bat.stats(&queries, &batches, &direct);
    printf("queries=%llu batches=%llu direct=%llu faceted_batches=%d max_faceted=%d oom=%d refused=%d checked=%d\n",
           (unsigned long long)queries, (unsigned long long)batches, (unsigned long long)direct, g_faceted_batches.load(),
           g_max_faceted.load(), g_oom.load(), refused.load(), g_checked.load());
    int bad = g_bad.load();
    if (g_faceted_batches.load() == 0 || refused.load() == 0 || direct != 0) bad++;
    if (g_oom.load() == 0 || g_max_faceted.load() > (int)OOM_ABOVE || batches >= queries) bad++;
    printf("wrong=%d bad=%d\n", wrong.load(), bad);
    return wrong.load() == 0 && bad == 0 ? 0 : 1;
}
