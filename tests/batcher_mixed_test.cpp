// Host-logic test of the mixed key of the micro-batching queue (oramacore_b200/csrc/batcher.h, OC_BATCHER_MIXED) with
// its own fake executor, which honours q_params.  Every request carries its id (the first component of its query vector
// and the term id of its one token); what it submitted is kept in g_desc[id].  The fake answers query i of a call from
// its id and its own scalars (q_params[i], or the call's scalars without q_params) into its row of p->limit entries,
// and records what each merged call held.  Many threads submit requests with random modes, limits, offsets,
// similarities, thresholds, vector limits and OMC arrays; the test checks that every caller gets exactly its own answer
// at its own limit, that requests with different scalars were merged (mixed) or never merged (default), that a merged
// call's stride is its largest limit and its requests share the route flags and the OMC arrays, and that requests the
// library would refuse for their scalars ran directly.  batcher_mixed_test mixed | default.
// Built and run by tests/test_batcher_mixed_host.py (g++, no CUDA).
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <random>
#include <thread>
#include <vector>

#include "../oramacore_b200/csrc/batcher.h"

static const uint32_t DIM = 4;
static const int MAX_IDS = 4000;
static const uint64_t OMC_A[2] = {3, 9}, OMC_B[3] = {1, 2, 5};
static const float MULT_A[2] = {2.f, 3.f}, MULT_B[3] = {1.5f, 2.5f, 0.5f};

struct Desc {
    int mode = OC_MODE_FULLTEXT;
    uint32_t limit = 0, offset = 0, vector_limit = 0;
    float similarity = 0.f, threshold = -1.f;
    int omc = 0;                       // 0: none, 1: OMC_A, 2: OMC_B
    bool direct = false;               // the library would refuse its scalars: it must run alone
};
static Desc g_desc[MAX_IDS];

// the answer of query `id` with scalars (limit, offset): n hits, then doc / score of hit j, and its count
static uint32_t n_of(uint32_t id, uint32_t limit) { return std::min<uint32_t>(limit, id % 37); }
static uint64_t doc_of(uint32_t id, uint32_t offset, uint32_t j) { return uint64_t(id) * 10000 + offset * 10 + j + 1; }
static float score_of(uint32_t id, int mode, float sim, float thr, uint32_t j) {
    return float(id) + float(mode) * 0.25f + sim + (thr >= 0.f ? 100.f : 0.f) - float(j) * 0.001f;
}
static uint64_t count_of(uint32_t id, uint32_t vl) { return uint64_t(id) * 3 + vl; }

std::atomic<int> g_bad{0};
std::atomic<uint32_t> g_merged{0}, g_mixed_calls{0}, g_omc_merged{0};

struct Fake {
    int operator()(const ocb::Call &c) const {
        const oc_search_params *p = c.p;
        if (c.kind != ocb::PLAIN) { g_bad++; return OC_ERR_INVALID; }
        const uint32_t B = p->n_queries, L = p->limit;
        const oc_query_params *qp = p->q_params;
        if (B > 1) g_merged++;
        bool differ = false, thr0 = false, deep0 = false;
        uint32_t max_limit = 0;
        for (uint32_t i = 0; i < B; i++) {
            const int mode = qp ? qp[i].mode : p->mode;
            uint32_t id;
            if (mode != OC_MODE_FULLTEXT) id = (uint32_t)llroundf(p->q_vecs[size_t(i) * DIM]);
            else id = p->term_id[p->token_term_offsets[p->q_token_offsets[i]]];
            if (id >= MAX_IDS) { g_bad++; return OC_ERR_INVALID; }
            const Desc &d = g_desc[id];
            const uint32_t limit = qp ? qp[i].limit : p->limit, offset = qp ? qp[i].offset : p->offset;
            const uint32_t vl = qp ? qp[i].vector_limit : p->vector_limit;
            const float sim = qp ? qp[i].similarity : p->similarity, thr = qp ? qp[i].threshold : p->threshold;
            // the scalars the library reads for query i are the ones its caller submitted
            if (mode != d.mode || limit != d.limit || offset != d.offset || vl != d.vector_limit || sim != d.similarity ||
                thr != d.threshold)
                g_bad++;
            if (B > 1 && d.direct) g_bad++;
            // a vector query's text and a fulltext query's vector are not carried
            if (qp && mode == OC_MODE_VECTOR && p->q_token_offsets && p->q_token_offsets[i + 1] != p->q_token_offsets[i]) g_bad++;
            if (qp && mode == OC_MODE_FULLTEXT && p->q_vecs && p->q_vecs[size_t(i) * DIM] != 0.f) g_bad++;
            // OMC: every query of a call submitted the call's arrays
            const uint64_t *od = d.omc == 1 ? OMC_A : d.omc == 2 ? OMC_B : nullptr;
            if ((od ? p->omc_doc_ids != od : p->n_omc != 0)) g_bad++;
            const bool thr_i = mode != OC_MODE_VECTOR && thr >= 0.f;
            const bool deep_i = mode != OC_MODE_FULLTEXT && (vl ? vl : limit) > ocb::TC_MAX_DEPTH;
            if (i == 0) { thr0 = thr_i; deep0 = deep_i; }
            else if (thr_i != thr0 || deep_i != deep0) g_bad++;   // the route flags are part of the key
            if (qp && i > 0 && (qp[i].mode != qp[0].mode || qp[i].limit != qp[0].limit || qp[i].offset != qp[0].offset)) differ = true;
            max_limit = std::max(max_limit, limit);
            if (limit > L) { g_bad++; return OC_ERR_INVALID; }
            const uint32_t n = n_of(id, limit);
            for (uint32_t j = 0; j < L; j++) {   // the row: n hits, then 0 (entries past the query's limit stay 0)
                c.docs[size_t(i) * L + j] = j < n ? doc_of(id, offset, j) : 0;
                c.scores[size_t(i) * L + j] = j < n ? score_of(id, mode, sim, thr, j) : 0.f;
            }
            c.n[i] = n;
            c.count[i] = count_of(id, vl);
        }
        if (qp && L != max_limit) g_bad++;           // the stride is the largest limit
        if (differ) g_mixed_calls++;
        if (B > 1 && p->n_omc) g_omc_merged++;
        return OC_OK;
    }
    int check(const oc_facets *, const oc_facet_req *, uint32_t) const { return OC_OK; }
};

int main(int argc, char **argv) {
    const bool mixed = argc > 1 && !strcmp(argv[1], "mixed");
    ocb::Batcher<Fake> q(Fake{}, DIM, 32, 2000, true, true, mixed);
    const int T = 16, PER = 60;
    std::mt19937 rng(7);
    // 24 scalar tuples, so that the default key also finds requests to merge
    Desc pool[24];
    for (Desc &d : pool) {
        d.mode = int(rng() % 3);
        d.limit = 1 + rng() % 60;
        d.offset = rng() % 41;
        d.similarity = float(rng() % 3) * 0.25f;
        d.threshold = rng() % 4 == 0 ? 0.5f : -1.f;
        d.vector_limit = rng() % 6 == 0 ? 129 + rng() % 40 : 0;   // deep: the exact sweep's route
    }
    for (int id = 0; id < T * PER; id++) {
        Desc &d = g_desc[id];
        d = pool[rng() % 24];
        d.omc = int(rng() % 3);
        if (rng() % 40 == 0) { d.offset = 1024; d.direct = mixed; }   // limit + offset > 1024: the library refuses it
    }
    {   // a request with its own q_params never joins a batch: the merged call's q_params are the requests' scalars
        float qv[DIM] = {1.f, 0.f, 0.f, 0.f};
        const oc_query_params e{OC_MODE_VECTOR, 5, 0, 0.f, -1.f, 0};
        oc_search_params p{};
        p.mode = OC_MODE_VECTOR; p.n_queries = 1; p.limit = 5; p.q_vecs = qv; p.q_params = &e;
        if (ocb::batchable(&p, true, true, false) || ocb::batchable(&p, true, true, true)) g_bad++;
        p.q_params = nullptr;
        if (!ocb::batchable(&p, true, true, false)) g_bad++;
    }
    std::atomic<int> wrong{0};
    std::vector<std::thread> th;
    for (int t = 0; t < T; t++)
        th.emplace_back([&, t] {
            for (int k = 0; k < PER; k++) {
                const uint32_t id = uint32_t(t * PER + k);
                const Desc &d = g_desc[id];
                float qv[DIM] = {float(id), 0.f, 0.f, 0.f};
                const uint32_t q_tok[2] = {0, 1}, tok_term[2] = {0, 1}, field = 0, term = id;
                const float w = 1.f;
                oc_search_params p{};
                p.mode = d.mode; p.n_queries = 1; p.limit = d.limit; p.offset = d.offset; p.similarity = d.similarity;
                p.threshold = d.threshold; p.bm25_k = 1.2f; p.bm25_b = 0.75f; p.vector_limit = d.vector_limit;
                p.q_vecs = qv; p.q_token_offsets = q_tok; p.token_term_offsets = tok_term; p.term_field = &field;
                p.term_id = &term; p.term_weight = &w;
                if (d.omc == 1) { p.omc_doc_ids = OMC_A; p.omc_mult = MULT_A; p.n_omc = 2; }
                if (d.omc == 2) { p.omc_doc_ids = OMC_B; p.omc_mult = MULT_B; p.n_omc = 3; }
                std::vector<uint64_t> docs(d.limit + 4, 77);   // 4 guard entries past the caller's limit
                std::vector<float> scores(d.limit + 4, 77.f);
                uint32_t n = 99; uint64_t cnt = 99;
                ocb::Request r{{ocb::PLAIN, &p, docs.data(), scores.data(), &n, &cnt}};
                const char *why = nullptr;
                const int rc = q.submit(r, &why);
                bool ok = rc == OC_OK && n == n_of(id, d.limit) && cnt == count_of(id, d.vector_limit);
                for (uint32_t j = 0; j < d.limit && ok; j++)
                    ok = docs[j] == (j < n ? doc_of(id, d.offset, j) : 0) &&
                         scores[j] == (j < n ? score_of(id, d.mode, d.similarity, d.threshold, j) : 0.f);
                for (uint32_t j = d.limit; j < d.limit + 4 && ok; j++) ok = docs[j] == 77 && scores[j] == 77.f;
                if (!ok) wrong++;
            }
        });
    for (auto &x : th) x.join();
    uint64_t nq = 0, nb = 0, nd = 0;
    q.stats(&nq, &nb, &nd);
    printf("queries=%llu batches=%llu direct=%llu merged_calls=%u mixed_calls=%u omc_merged=%u\n", (unsigned long long)nq,
           (unsigned long long)nb, (unsigned long long)nd, g_merged.load(), g_mixed_calls.load(), g_omc_merged.load());
    printf("wrong=%d bad=%d\n", wrong.load(), g_bad.load());
    if (wrong || g_bad) return 1;
    if (g_merged == 0) return 2;                                  // requests were coalesced
    if (mixed && (g_mixed_calls == 0 || g_omc_merged == 0)) return 3;   // different scalars and OMC requests shared calls
    if (!mixed && (g_mixed_calls != 0 || g_omc_merged != 0)) return 4;  // the default key keeps them apart
    return 0;
}
