// Host-logic test of where programs in the micro-batching queue (oramacore_b200/csrc/batcher.h) with a fake executor.
// Every request carries its id (the term id of its one token); what it submitted is kept in g_desc[id]: a where program
// (a few nodes, polygons with their own vertices), a device filter handle (p->filter), or neither.  The fake checks, per
// query of each call, that a merged call with a program carries q_where and no q_filters, that each query's nodes are its
// request's with polygon vertices rebased onto the merged arrays, that a handle request became one FILTER node and an
// unfiltered one an empty range; and that a call in which no request has a program still carries q_filters (or nothing)
// as before.  batcher_where_test programs | handles.
// Built and run by tests/test_batcher_where_host.py (g++, no CUDA).
#include <atomic>
#include <cstdio>
#include <cstring>
#include <random>
#include <thread>
#include <vector>

#include "../oramacore_b200/csrc/batcher.h"

static const int MAX_IDS = 4000;
static char g_handles[8];   // fake oc_filter handles: their addresses

struct Desc {
    int kind = 0;                          // 0 none, 1 program, 2 handle
    std::vector<oc_where_node> nodes;      // first_vertex indexes lat / lon below
    std::vector<double> lat, lon;
    oc_where where{};
    uint32_t off[2] = {0, 0};
    const oc_filter *filter = nullptr;
};
static Desc g_desc[MAX_IDS];

std::atomic<int> g_bad{0};
std::atomic<uint32_t> g_merged{0}, g_merged_where{0}, g_merged_handles{0};

static bool same_node(const oc_where_node &a, const oc_where_node &b) {
    return a.op == b.op && a.field == b.field && a.arg == b.arg && a.n_vertices == b.n_vertices && a.a == b.a && a.src == b.src;
}

struct Fake {
    int operator()(const ocb::Call &c) const {
        const oc_search_params *p = c.p;
        const uint32_t B = p->n_queries;
        if (B > 1) g_merged++;
        bool any_prog = false, any_handle = false;
        for (uint32_t i = 0; i < B; i++) {
            const uint32_t id = p->term_id[p->token_term_offsets[p->q_token_offsets[i]]];
            if (id >= MAX_IDS) { g_bad++; return OC_ERR_INVALID; }
            const Desc &d = g_desc[id];
            any_prog = any_prog || d.kind == 1;
            any_handle = any_handle || d.kind == 2;
        }
        if (B > 1 && any_prog) g_merged_where++;
        if (B > 1 && any_handle && !any_prog) g_merged_handles++;
        for (uint32_t i = 0; i < B; i++) {
            const uint32_t id = p->term_id[p->token_term_offsets[p->q_token_offsets[i]]];
            const Desc &d = g_desc[id];
            if (any_prog) {
                const oc_where *w = p->q_where;
                if (!w || p->q_filters || p->filter) { g_bad++; continue; }
                const uint32_t o0 = w->q_node_offsets[i], o1 = w->q_node_offsets[i + 1];
                if (d.kind == 0 && o1 != o0) g_bad++;
                if (d.kind == 2 && (o1 != o0 + 1 || w->nodes[o0].op != OC_WHERE_FILTER || w->nodes[o0].src != d.filter)) g_bad++;
                if (d.kind == 1) {
                    if (o1 - o0 != d.nodes.size()) { g_bad++; continue; }
                    for (uint32_t k = 0; k < o1 - o0; k++) {
                        const oc_where_node &m = w->nodes[o0 + k], &s = d.nodes[k];
                        if (!same_node(m, s)) g_bad++;
                        if (s.op == OC_WHERE_GEO_POLYGON)
                            for (uint32_t v = 0; v < s.n_vertices; v++)
                                if (w->vertex_lat[m.first_vertex + v] != d.lat[s.first_vertex + v] ||
                                    w->vertex_lon[m.first_vertex + v] != d.lon[s.first_vertex + v])
                                    g_bad++;
                    }
                }
            } else {   // no program: q_filters exactly as before
                if (p->q_where) g_bad++;
                if (p->filter) g_bad++;
                if (any_handle && (!p->q_filters || p->q_filters[i] != d.filter)) g_bad++;
                if (!any_handle && p->q_filters) g_bad++;
            }
        }
        for (uint32_t i = 0; i < B; i++) {
            const uint32_t id = p->term_id[p->token_term_offsets[p->q_token_offsets[i]]];
            c.n[i] = 1;
            c.docs[size_t(i) * p->limit] = uint64_t(id) * 10 + 1;
            c.scores[size_t(i) * p->limit] = float(id);
            c.count[i] = id;
        }
        return OC_OK;
    }
    int check(const oc_facets *, const oc_facet_req *, uint32_t) const { return OC_OK; }
};

static void make_desc(int id, std::mt19937 &rng, bool programs) {
    Desc &d = g_desc[id];
    d.kind = programs ? int(rng() % 3) : (rng() % 2 ? 2 : 0);
    if (d.kind == 2) d.filter = reinterpret_cast<const oc_filter *>(&g_handles[rng() % 8]);
    if (d.kind != 1) return;
    const void *store = &g_handles[0];
    auto leaf = [&](uint32_t op) {
        oc_where_node n{};
        n.op = op; n.field = rng() % 5; n.arg = rng() % 2; n.a = double(id) + 0.5; n.src = store;
        if (op == OC_WHERE_GEO_POLYGON) {
            n.first_vertex = (uint32_t)d.lat.size(); n.n_vertices = 3 + rng() % 3;
            for (uint32_t v = 0; v < n.n_vertices; v++) { d.lat.push_back(id + v * 0.01); d.lon.push_back(-double(id) - v); }
        }
        d.nodes.push_back(n);
    };
    const uint32_t k = 1 + rng() % 3;
    for (uint32_t j = 0; j < k; j++) leaf(j % 2 ? OC_WHERE_GEO_POLYGON : OC_WHERE_RANGE);
    if (k > 1) { oc_where_node n{}; n.op = OC_WHERE_AND; n.arg = k; d.nodes.push_back(n); }
    d.off[1] = (uint32_t)d.nodes.size();
    d.where = oc_where{1000, d.off, d.nodes.data(), d.lat.empty() ? nullptr : d.lat.data(), d.lon.empty() ? nullptr : d.lon.data()};
}

int main(int argc, char **argv) {
    const bool programs = argc > 1 && strcmp(argv[1], "programs") == 0;
    const int T = 16, PER = 120;
    std::mt19937 rng(7);
    for (int id = 0; id < T * PER; id++) make_desc(id, rng, programs);
    ocb::Batcher<Fake> q(Fake{}, 4, 32, 2000, false, true, false);
    std::atomic<int> wrong{0};
    std::vector<std::thread> ts;
    for (int t = 0; t < T; t++)
        ts.emplace_back([&, t] {
            for (int r = 0; r < PER; r++) {
                const uint32_t id = uint32_t(t * PER + r);
                const Desc &d = g_desc[id];
                uint32_t qoff[2] = {0, 1}, toff[2] = {0, 1}, field = 0, term = id;
                float w = 1.f;
                oc_search_params p{};
                p.mode = OC_MODE_FULLTEXT; p.n_queries = 1; p.limit = 4; p.bm25_k = 1.2f; p.bm25_b = 0.75f; p.threshold = -1.f;
                p.q_token_offsets = qoff; p.token_term_offsets = toff; p.term_field = &field; p.term_id = &term; p.term_weight = &w;
                p.filter = d.filter;
                if (d.kind == 1) p.q_where = &d.where;
                uint64_t docs[4] = {}, count = 0;
                float scores[4] = {};
                uint32_t n = 0;
                ocb::Request req{{ocb::PLAIN, &p, docs, scores, &n, &count}};
                const char *why = nullptr;
                const int rc = q.submit(req, &why);
                if (rc != OC_OK || n != 1 || docs[0] != uint64_t(id) * 10 + 1 || count != id) wrong++;
            }
        });
    for (auto &t : ts) t.join();
    uint64_t nq = 0, nb = 0, nd = 0;
    q.stats(&nq, &nb, &nd);
    int bad = g_bad.load();
    if (g_merged == 0) bad++;
    if (programs && g_merged_where == 0) bad++;
    if (!programs && g_merged_handles == 0) bad++;
    printf("queries=%llu batches=%llu direct=%llu merged=%u where=%u handles=%u\n", (unsigned long long)nq,
           (unsigned long long)nb, (unsigned long long)nd, g_merged.load(), g_merged_where.load(), g_merged_handles.load());
    printf("wrong=%d bad=%d\n", wrong.load(), bad);
    return wrong || bad ? 1 : 0;
}
