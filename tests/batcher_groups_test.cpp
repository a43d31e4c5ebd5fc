// Host-logic test of grouped requests in the micro-batching queue (oramacore_b200/csrc/batcher.h) with fake executors:
// 12 threads submit single queries through submit() (plain) and submit_groups() (a groupBy handle of 1, 3 or 7 groups
// or none, max_results 0-10, a sort or score order, 0-2 promote items, a group stride of its need plus 0-3).  It checks
// that
//   - grouped and plain requests never share a batch, and grouped requests do coalesce;
//   - the grouped executor sees each request's handle, max_results, sort and items at its own position and a group
//     stride no smaller than any request's need, and each caller gets back its own rows at its own stride, with
//     differing n_groups and strides inside one batch;
//   - a merged call that fails with OC_ERR_OOM (here: any batch of more than 5 requests) is split in halves and every
//     request still succeeds;
//   - a request the merged call would refuse (max_results > OC_MAX_TOPK) runs alone and gets the refusal, and the
//     requests around it succeed;
//   - a request with a group stride below its need is refused with OC_ERR_INVALID and never reaches an executor.
// Built and run by tests/test_batcher_groups_host.py (g++, no CUDA).
#include <atomic>
#include <cmath>
#include <cstdio>
#include <random>
#include <thread>
#include <vector>

#include "../oramacore_b200/csrc/batcher.h"

static const uint32_t DIM = 4, LIMIT = 3, OOM_ABOVE = 5;
static const int N_GB = 3, N_FIELDS = 2;
static const uint64_t GB_GROUPS[N_GB] = {1, 3, 7};
static char g_gb[N_GB], g_fields[N_FIELDS];   // fake handles: only their addresses are used
static const oc_group_by *gb(int i) { return reinterpret_cast<const oc_group_by *>(&g_gb[i]); }
static const oc_sort_field *field(int i) { return reinterpret_cast<const oc_sort_field *>(&g_fields[i]); }
static const int T = 12, Q = 150, N_IDS = T * Q;

// what every request carries, drawn once per id
struct Req {
    bool plain = false, invalid = false, oversized = false;
    int gb = -1;                        // -1: no groups
    uint32_t m = 0, k = 0, stride = 0;  // max_results, items, its group stride
    int field = -1, order = 0;
};
static Req g_req[N_IDS];
static uint32_t need_of(const Req &r) { return r.gb < 0 ? 0 : r.k ? 2 * r.m + r.k : r.m; }
// the rows the fake library writes: row g of query id has n = (id + g) % (need + 1) entries
static uint32_t n_of(uint32_t id, uint64_t g) { return uint32_t((id + g) % (need_of(g_req[id]) + 1)); }
static uint64_t doc_of(uint32_t id, uint64_t g, uint32_t j) { return uint64_t(id) * 100000 + g * 100 + j + 1; }

std::atomic<int> g_bad{0}, g_grouped_batches{0}, g_oom{0}, g_max_grouped{0};
static uint32_t id_of(const oc_search_params *p, uint32_t i) { return (uint32_t)llround(p->q_vecs[size_t(i) * DIM]); }

struct FakeExec {
    int operator()(const oc_search_params *p, uint64_t *docs, float *, uint32_t *n, uint64_t *count) const {
        for (uint32_t i = 0; i < p->n_queries; i++) {
            const uint32_t id = id_of(p, i);
            if (id >= (uint32_t)N_IDS || !g_req[id].plain) { g_bad++; continue; }   // a grouped request in a plain batch
            docs[size_t(i) * p->limit] = id; n[i] = 1; count[i] = id;
        }
        return 0;
    }
};
struct FakeGroupedExec {
    int operator()(const oc_search_params *p, const oc_group_req *q, const oc_pins *pins, uint32_t stride, uint64_t *docs,
                   float *, double *, uint32_t *n, uint64_t *count, float *, uint8_t *, uint64_t *g_doc, float *g_score,
                   double *g_values, uint32_t *g_n) const {
        const uint32_t B = p->n_queries;
        for (uint32_t i = 0; i < B; i++)
            if (q[i].max_results > OC_MAX_TOPK) return OC_ERR_UNSUPPORTED;
        if (B > OOM_ABOVE) { g_oom++; return OC_ERR_OOM; }
        if (B > 1) {
            g_grouped_batches++;
            int prev = g_max_grouped.load();
            while ((int)B > prev && !g_max_grouped.compare_exchange_weak(prev, (int)B)) {}
        }
        uint64_t row = 0;
        for (uint32_t i = 0; i < B; i++) {
            const uint32_t id = id_of(p, i);
            if (id >= (uint32_t)N_IDS) { g_bad++; return OC_ERR_INVALID; }
            const Req &r = g_req[id];
            const uint32_t k = pins ? pins->q_pin_offsets[i + 1] - pins->q_pin_offsets[i] : 0;
            const bool same = !r.plain && !r.invalid && (r.gb < 0 ? q[i].groups == nullptr : q[i].groups == gb(r.gb)) &&
                              q[i].max_results == r.m && k == r.k && stride >= need_of(r) &&
                              (r.field < 0 ? q[i].sort.field == nullptr : q[i].sort.field == field(r.field) && q[i].sort.order == r.order);
            if (!same) g_bad++;
            for (uint32_t j = 0; j < k; j++)
                if (pins->doc_ids[pins->q_pin_offsets[i] + j] != uint64_t(id) * 10 + j) g_bad++;
            docs[size_t(i) * p->limit] = id; n[i] = 1; count[i] = id;
            const uint64_t G = r.gb < 0 ? 0 : GB_GROUPS[r.gb];
            for (uint64_t g = 0; g < G; g++, row++) {
                g_n[row] = n_of(id, g);
                for (uint32_t j = 0; j < stride; j++) {
                    const bool in = j < g_n[row];
                    g_doc[row * stride + j] = in ? doc_of(id, g, j) : 0;
                    g_score[row * stride + j] = in ? float(j) : 0.f;
                    g_values[row * stride + j] = in ? double(id) + 0.5 : 0.0;
                }
            }
        }
        return 0;
    }
};

int main() {
    std::mt19937 rng(7);
    for (int id = 0; id < N_IDS; id++) {
        Req &r = g_req[id];
        const int kind = int(rng() % 20);
        r.plain = kind < 4;
        r.invalid = kind == 4;
        r.oversized = kind == 5;
        if (r.plain) continue;
        r.gb = int(rng() % (N_GB + 1)) - 1;
        if (r.gb < 0 && kind == 5) r.gb = 0;
        r.m = r.oversized ? OC_MAX_TOPK + 1 : uint32_t(rng() % 11);
        r.k = uint32_t(rng() % 3);
        if (r.oversized) r.k = 0;
        r.field = int(rng() % (N_FIELDS + 1)) - 1;
        r.order = int(rng() % 2);
        r.stride = need_of(r) + uint32_t(rng() % 4);
        if (r.invalid) { r.gb = 1; r.m = 4; r.stride = need_of(r) - 1; }
    }
    ocb::Batcher<FakeExec, ocb::NoSortedExec, FakeGroupedExec> bat(FakeExec{}, DIM, 32, 2000, true, false);
    std::atomic<int> wrong{0}, refused{0}, oversized_refused{0};
    auto worker = [&](int t) {
        for (int id = t; id < N_IDS; id += T) {
            const Req &r = g_req[id];
            float qv[DIM] = {float(id), 0, 0, 0};
            oc_search_params p{};
            p.mode = OC_MODE_VECTOR; p.n_queries = 1; p.limit = LIMIT; p.q_vecs = qv;
            std::vector<uint64_t> docs(LIMIT, 7);
            std::vector<float> scores(LIMIT, 7.f);
            uint32_t n = 7;
            uint64_t count = 7;
            if (r.plain) {
                const int rc = bat.submit(&p, docs.data(), scores.data(), &n, &count);
                if (rc != 0 || docs[0] != uint64_t(id) || n != 1 || count != uint64_t(id)) wrong++;
                continue;
            }
            const oc_group_req req{r.gb < 0 ? nullptr : gb(r.gb), r.m, oc_sort{r.field < 0 ? nullptr : field(r.field), r.order}};
            std::vector<uint32_t> off = {0, r.k};
            std::vector<uint64_t> pdoc(std::max<uint32_t>(r.k, 1));
            std::vector<uint32_t> ppos(std::max<uint32_t>(r.k, 1), 0);
            for (uint32_t j = 0; j < r.k; j++) pdoc[j] = uint64_t(id) * 10 + j;
            const oc_pins pins{off.data(), pdoc.data(), ppos.data(), 1};
            const uint64_t G = r.gb < 0 ? 0 : GB_GROUPS[r.gb];
            const size_t cells = std::max<size_t>(G * r.stride, 1);
            std::vector<uint64_t> gd(cells, 7);
            std::vector<float> gs(cells, 7.f);
            std::vector<double> gv(cells, 7.0), sv(LIMIT, 7.0);
            std::vector<uint32_t> gn(std::max<uint64_t>(G, 1), 7);
            std::vector<float> ps(2, 7.f);
            std::vector<uint8_t> pp(2, 7);
            const int rc = bat.submit_groups(&p, &req, G, &pins, r.stride, docs.data(), scores.data(), sv.data(), &n, &count,
                                             ps.data(), pp.data(), gd.data(), gs.data(), gv.data(), gn.data());
            if (r.invalid) {
                if (rc != OC_ERR_INVALID || gd[0] != 7 || gn[0] != 7 || n != 7) wrong++;
                refused++;
                continue;
            }
            if (r.oversized) {
                if (rc != OC_ERR_UNSUPPORTED || n != 7) wrong++;
                oversized_refused++;
                continue;
            }
            if (rc != 0 || docs[0] != uint64_t(id) || n != 1 || count != uint64_t(id)) { wrong++; continue; }
            for (uint64_t g = 0; g < G; g++) {
                const uint32_t gn_want = n_of(id, g);
                if (gn[g] != gn_want) wrong++;
                for (uint32_t j = 0; j < r.stride; j++) {
                    const bool in = j < gn_want;
                    const size_t o = g * r.stride + j;
                    if (gd[o] != (in ? doc_of(id, g, j) : 0) || gs[o] != (in ? float(j) : 0.f) || gv[o] != (in ? double(id) + 0.5 : 0.0))
                        wrong++;
                }
            }
        }
    };
    std::vector<std::thread> th;
    for (int t = 0; t < T; t++) th.emplace_back(worker, t);
    for (auto &x : th) x.join();
    uint64_t queries = 0, batches = 0, direct = 0;
    bat.stats(&queries, &batches, &direct);
    printf("queries=%llu batches=%llu direct=%llu grouped_batches=%d max_grouped=%d oom=%d refused=%d oversized=%d\n",
           (unsigned long long)queries, (unsigned long long)batches, (unsigned long long)direct, g_grouped_batches.load(),
           g_max_grouped.load(), g_oom.load(), refused.load(), oversized_refused.load());
    int bad = g_bad.load();
    if (g_grouped_batches.load() == 0 || refused.load() == 0 || oversized_refused.load() == 0) bad++;
    if (g_oom.load() == 0 || g_max_grouped.load() > (int)OOM_ABOVE || batches >= queries) bad++;
    printf("wrong=%d bad=%d\n", wrong.load(), bad);
    return wrong.load() == 0 && bad == 0 ? 0 : 1;
}
