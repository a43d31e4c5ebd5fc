// dict.h — native term dictionary + batch query-term resolution (host only, no CUDA).
//
// What the reference does on the host before the posting walk (SURVEY.md §8f-3):
//   * TextParser::tokenize_and_stem(term) -> [(original, [stems])]; exact => originals only, else
//     originals + stems flattened; no token at all => [""] (token_score.rs:196-209);
//   * per string field, StringStorage expands every token to index terms through its FST
//     (string_field.rs:208-225): exact term when `exact` (tolerance Some(0), token_score.rs:240), terms
//     within Levenshtein distance t when tolerance = Some(t) (fulltext_search.rs:956-1018), prefix
//     expansion otherwise ("christoph" matches "Christopher", fulltext_search.rs:633-644); an exactly
//     matching term carries the exact-match boost (boost_integration.rs:449-490).
// This file provides that step natively so a 256-query batch resolves in tens of microseconds instead of
// a Python scan of the vocabulary: per field a dictionary with STABLE term ids (ids are what
// oc_str_insert / the posting lists use; new terms get the next id) plus a lexicographically sorted index
// with an LCP array: prefix expansion = two binary searches, bounded Levenshtein = one walk over the sorted
// terms that shares the DP rows of common prefixes and prunes whole prefix subtrees.
// Output = the CSR arrays oc_search takes (q_token_offsets / token_term_offsets / term_field / term_id /
// term_weight).  Within a token the terms are emitted field by field in lexicographic order, so the BM25F
// summation order — and with it every score bit — is a function of the dictionary content only.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <functional>
#include <mutex>
#include <shared_mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

namespace ocd {

// oc_stem_fn: writes the stem of tok[0..len) into out (cap bytes), returns its length; 0 = no stem.
typedef size_t (*StemFn)(const char *tok, size_t len, char *out, size_t cap, void *user);

// lower-case ASCII alphanumeric runs (the stand-in tokenizer of the parity tests; a host NLP stack can
// pre-tokenise instead and pass one token per "text")
inline void tokenize(const char *text, std::vector<std::string> &out) {
    std::string cur;
    for (const unsigned char *p = reinterpret_cast<const unsigned char *>(text); *p; ++p) {
        unsigned char ch = *p;
        if (ch >= 'A' && ch <= 'Z') ch = (unsigned char)(ch - 'A' + 'a');
        if ((ch >= 'a' && ch <= 'z') || (ch >= '0' && ch <= '9')) cur.push_back((char)ch);
        else if (!cur.empty()) { out.push_back(cur); cur.clear(); }
    }
    if (!cur.empty()) out.push_back(cur);
}

struct FieldDict {
    std::vector<std::string> terms;                    // id -> term
    std::unordered_map<std::string, uint32_t> ids;     // term -> id
    std::vector<uint32_t> sorted;                      // ids in lexicographic (byte) order of their terms
    std::vector<uint32_t> lcp;                         // lcp[i] = common prefix of sorted[i-1], sorted[i] (lcp[0] = 0)
    std::vector<uint32_t> next_smaller;                // next_smaller[i] = first j > i with lcp[j] < lcp[i] (or size): subtree skips
    size_t n_indexed = 0;                              // terms[0..n_indexed) are in `sorted`

    uint32_t add(const std::string &t) {
        auto it = ids.find(t);
        if (it != ids.end()) return it->second;
        const uint32_t id = (uint32_t)terms.size();
        terms.push_back(t);
        ids.emplace(t, id);
        return id;
    }
    bool stale() const { return n_indexed != terms.size(); }
    void reindex() {   // merge the unsorted tail into the sorted index, rebuild the LCP array
        if (!stale()) return;
        const size_t old = sorted.size();
        for (size_t i = n_indexed; i < terms.size(); i++) sorted.push_back((uint32_t)i);
        auto less = [&](uint32_t a, uint32_t b) { return terms[a] < terms[b]; };
        std::sort(sorted.begin() + old, sorted.end(), less);
        std::inplace_merge(sorted.begin(), sorted.begin() + old, sorted.end(), less);
        n_indexed = terms.size();
        lcp.assign(sorted.size(), 0);
        for (size_t i = 1; i < sorted.size(); i++) {
            const std::string &a = terms[sorted[i - 1]], &b = terms[sorted[i]];
            uint32_t l = 0;
            const uint32_t m = (uint32_t)std::min(a.size(), b.size());
            while (l < m && a[l] == b[l]) l++;
            lcp[i] = l;
        }
        // every position in (i, next_smaller[i]) has lcp >= lcp[i]: the end of a prefix subtree is reached in at
        // most (term length) hops instead of a linear walk
        next_smaller.assign(sorted.size(), (uint32_t)sorted.size());
        std::vector<uint32_t> st;
        for (size_t i = 0; i < sorted.size(); i++) {
            while (!st.empty() && lcp[st.back()] > lcp[i]) { next_smaller[st.back()] = (uint32_t)i; st.pop_back(); }
            st.push_back((uint32_t)i);
        }
    }
    // [lo, hi) of sorted positions whose term starts with `p`
    void prefix_range(const std::string &p, size_t *lo, size_t *hi) const {
        auto cmp_lo = [&](uint32_t id, const std::string &key) { return terms[id].compare(0, key.size(), key) < 0; };
        const auto b = std::lower_bound(sorted.begin(), sorted.end(), p, cmp_lo);
        auto cmp_hi = [&](const std::string &key, uint32_t id) { return terms[id].compare(0, key.size(), key) > 0; };
        const auto e = std::upper_bound(b, sorted.end(), p, cmp_hi);
        *lo = size_t(b - sorted.begin());
        *hi = size_t(e - sorted.begin());
    }
};

struct Resolved {   // CSR arrays for oc_search
    std::vector<uint32_t> q_token_offsets{0}, token_term_offsets{0}, term_field, term_id;
    std::vector<float> term_weight;
};

struct ResolveOpts {
    bool exact = false;
    int tolerance = -1;                 // < 0: none (prefix expansion)
    const float *field_boost = nullptr; // per field, NULL = 1.0
    const uint8_t *field_mask = nullptr;// per field (properties), NULL = all
    float exact_match_boost = 2.0f;
};

// A (token, field) expansion with tolerance >= 1 that resolve_q hands to a FuzzyRun (the device): the sorted positions
// of `field` whose term starts with tok or lies within byte-wise Levenshtein distance t of it, ascending — what
// Dict::fuzzy emits.  Tokens longer than one 64-bit pattern word stay with the host walk.
constexpr size_t FUZZY_RUN_MAX_TOK = 64;
struct FuzzyPair { uint32_t field, t; const std::string *tok; };
// pair i's terms are id[off[i] .. off[i+1]) in emission order; exact[e]: the term equals the token
struct FuzzyLists { std::vector<uint32_t> off, id; std::vector<uint8_t> exact; };
// runs the pairs over fields[] (held under the dictionary's shared lock); gen = Dict::generation().  Returns 0 or an
// error code, which resolve_q passes on.
typedef std::function<int(const std::vector<FieldDict> &fields, uint64_t gen, const std::vector<FuzzyPair> &pairs,
                          FuzzyLists *out)> FuzzyRun;

class Dict {
public:
    explicit Dict(uint32_t n_fields) : fields_(n_fields) {}
    uint32_t n_fields() const { return (uint32_t)fields_.size(); }

    void add_terms(uint32_t field, const char *const *terms, uint32_t n, uint32_t *out_ids) {
        std::unique_lock<std::shared_mutex> g(mu_);
        FieldDict &f = fields_[field];
        const size_t before = f.terms.size();
        for (uint32_t i = 0; i < n; i++) {
            const uint32_t id = f.add(terms[i]);
            if (out_ids) out_ids[i] = id;
        }
        if (f.terms.size() != before) gen_++;
    }
    bool lookup(uint32_t field, const char *term, uint32_t *id) {
        std::shared_lock<std::shared_mutex> g(mu_);
        const FieldDict &f = fields_[field];
        auto it = f.ids.find(term);
        if (it == f.ids.end()) return false;
        *id = it->second;
        return true;
    }
    uint32_t size(uint32_t field) {
        std::shared_lock<std::shared_mutex> g(mu_);
        return (uint32_t)fields_[field].terms.size();
    }
    void set_stemmer(StemFn fn, void *user) { std::unique_lock<std::shared_mutex> g(mu_); stem_ = fn; stem_user_ = user; }

    // bumped by add_terms (a new term) and by the reindex of a resolve; read under the shared lock (FuzzyRun)
    uint64_t generation() const { return gen_; }

    void resolve(const char *const *texts, uint32_t n_queries, const ResolveOpts &o, Resolved *out) {
        resolve_q(texts, n_queries, std::vector<ResolveOpts>(n_queries, o), nullptr, out);
    }
    // Query q with its own opts[q].  With `run`, every (token, field) pair of a query with tolerance >= 1 whose token
    // fits FUZZY_RUN_MAX_TOK is expanded by run, everything else here; the output is the same either way.  A failing
    // run's code is returned and `out` is left as it was.
    int resolve_q(const char *const *texts, uint32_t n_queries, const std::vector<ResolveOpts> &opts, const FuzzyRun *run,
                  Resolved *out) {
        {   // bring the sorted indexes up to date (exclusive), then resolve under the shared lock
            bool need = false;
            { std::shared_lock<std::shared_mutex> g(mu_); for (auto &f : fields_) need = need || f.stale(); }
            if (need) { std::unique_lock<std::shared_mutex> g(mu_); for (auto &f : fields_) f.reindex(); gen_++; }
        }
        std::shared_lock<std::shared_mutex> g(mu_);
        std::vector<Plan> per(n_queries);
        auto work = [&](uint32_t q0, uint32_t q1) { for (uint32_t q = q0; q < q1; q++) plan_one(texts[q], opts[q], run != nullptr, &per[q]); };
        // the bounded-Levenshtein walk is the only expensive mode: without a FuzzyRun, spread its queries over the host cores
        bool walk = false;
        for (const ResolveOpts &o : opts) walk = walk || (!o.exact && o.tolerance >= 0);
        unsigned nt = 1;
        if (!run && walk && n_queries >= 8) nt = std::min<unsigned>(std::max(1u, std::thread::hardware_concurrency()), std::min<unsigned>(n_queries / 4, 32));
        if (nt <= 1) work(0, n_queries);
        else {
            std::vector<std::thread> th;
            for (unsigned t = 0; t < nt; t++) th.emplace_back(work, uint32_t(uint64_t(n_queries) * t / nt), uint32_t(uint64_t(n_queries) * (t + 1) / nt));
            for (auto &t : th) t.join();
        }
        std::vector<FuzzyPair> pairs;
        std::vector<uint32_t> pair0(n_queries);
        for (uint32_t q = 0; q < n_queries; q++) {
            pair0[q] = (uint32_t)pairs.size();
            for (auto &d : per[q].dev) pairs.push_back({d.second, (uint32_t)opts[q].tolerance, &per[q].toks[d.first]});
        }
        FuzzyLists dev;
        if (!pairs.empty()) {
            const int rc = (*run)(fields_, gen_, pairs, &dev);
            if (rc) return rc;
        }
        size_t n_tok = 0, n_term = dev.id.size();
        for (auto &p : per) { n_tok += p.toks.size(); n_term += p.id.size(); }
        out->q_token_offsets.assign(1, 0u); out->token_term_offsets.assign(1, 0u);
        out->q_token_offsets.reserve(n_queries + 1); out->token_term_offsets.reserve(n_tok + 1);
        out->term_field.clear(); out->term_id.clear(); out->term_weight.clear();
        out->term_field.reserve(n_term); out->term_id.reserve(n_term); out->term_weight.reserve(n_term);
        for (uint32_t q = 0; q < n_queries; q++) {
            const Plan &p = per[q];
            const ResolveOpts &o = opts[q];
            size_t s = 0;
            for (uint32_t k = 0; k < p.toks.size(); k++) {
                for (; s < p.segs.size() && p.segs[s].tok == k; s++) {
                    const Plan::Seg &sg = p.segs[s];
                    const float w = o.field_boost ? o.field_boost[sg.field] : 1.0f;
                    const uint32_t *ids = p.id.data() + sg.h0;
                    const uint8_t *ex = p.exact.data() + sg.h0;
                    size_t n = sg.h1 - sg.h0;
                    if (sg.dev != Plan::HOST) {
                        const uint32_t i = pair0[q] + sg.dev;
                        ids = dev.id.data() + dev.off[i]; ex = dev.exact.data() + dev.off[i]; n = dev.off[i + 1] - dev.off[i];
                    }
                    for (size_t e = 0; e < n; e++) {
                        out->term_field.push_back(sg.field); out->term_id.push_back(ids[e]);
                        out->term_weight.push_back(ex[e] ? w * o.exact_match_boost : w);
                    }
                }
                out->token_term_offsets.push_back((uint32_t)out->term_id.size());
            }
            out->q_token_offsets.push_back((uint32_t)out->token_term_offsets.size() - 1);
        }
        return 0;
    }

private:
    // one query's expansion before the FuzzyRun lists are in: per (token, field), in token then field order, either
    // host-expanded terms or a pair for the run
    struct Plan {
        static constexpr uint32_t HOST = 0xffffffffu;
        struct Seg { uint32_t tok, field, dev, h0, h1; };   // dev: the query's run pair, or HOST: terms [h0, h1) below
        std::vector<std::string> toks;
        std::vector<Seg> segs;
        std::vector<uint32_t> id;
        std::vector<uint8_t> exact;
        std::vector<std::pair<uint32_t, uint32_t>> dev;     // run pairs: (token, field)
    };
    // token_score.rs:196-209: originals (+ stems unless exact); nothing => [""]
    void query_tokens(const char *text, bool exact, std::vector<std::string> &toks) const {
        std::vector<std::string> orig;
        tokenize(text, orig);
        for (auto &t : orig) {
            toks.push_back(t);
            if (!exact && stem_) {
                char buf[256];
                const size_t n = stem_(t.data(), t.size(), buf, sizeof(buf), stem_user_);
                if (n && n <= sizeof(buf) && std::string(buf, n) != t) toks.emplace_back(buf, n);
            }
        }
        if (toks.empty()) toks.emplace_back("");
    }
    void plan_one(const char *text, const ResolveOpts &o, bool run, Plan *p) const {
        query_tokens(text, o.exact, p->toks);
        for (uint32_t k = 0; k < p->toks.size(); k++) {
            const std::string &tok = p->toks[k];
            for (uint32_t fi = 0; fi < fields_.size(); fi++) {
                if (o.field_mask && !o.field_mask[fi]) continue;
                if (run && !o.exact && o.tolerance >= 1 && tok.size() <= FUZZY_RUN_MAX_TOK) {
                    p->segs.push_back({k, fi, (uint32_t)p->dev.size(), 0, 0});
                    p->dev.emplace_back(k, fi);
                    continue;
                }
                const FieldDict &f = fields_[fi];
                const uint32_t h0 = (uint32_t)p->id.size();
                auto emit = [&](uint32_t id, bool is_exact) { p->id.push_back(id); p->exact.push_back(is_exact); };
                if (o.exact) {
                    auto it = f.ids.find(tok);
                    if (it != f.ids.end()) emit(it->second, true);
                } else if (o.tolerance < 0) {
                    size_t lo, hi;
                    f.prefix_range(tok, &lo, &hi);
                    for (size_t i = lo; i < hi; i++) emit(f.sorted[i], f.terms[f.sorted[i]].size() == tok.size());
                } else {
                    fuzzy(f, tok, (uint32_t)o.tolerance, emit);
                }
                p->segs.push_back({k, fi, Plan::HOST, h0, (uint32_t)p->id.size()});
            }
        }
    }
    // terms within Levenshtein distance t of tok, plus the terms tok is a prefix of, in lexicographic order.
    // One pass over the sorted terms: DP row d (distance of term[0..d) to every prefix of tok) is shared by
    // all terms with that prefix; when the whole row exceeds t no extension can come back under it, so the
    // subtree of that prefix is skipped through the LCP array.
    template <class Emit>
    static void fuzzy(const FieldDict &f, const std::string &tok, uint32_t t, Emit emit) {
        const size_t V = f.sorted.size(), m = tok.size();
        size_t plo, phi;
        f.prefix_range(tok, &plo, &phi);
        std::vector<std::vector<uint32_t>> dp(1, std::vector<uint32_t>(m + 1));
        for (size_t j = 0; j <= m; j++) dp[0][j] = (uint32_t)j;
        size_t valid = 0;   // dp rows 0..valid hold the prefix of the previous visited term
        size_t i = 0;
        uint32_t carry = 0xffffffffu;   // min lcp over positions skipped since the last visited term
        while (i < V) {
            if (i == plo && phi > plo) {   // prefix matches: no DP needed
                for (size_t k = plo; k < phi; k++) {
                    emit(f.sorted[k], f.terms[f.sorted[k]].size() == m);
                    carry = std::min(carry, f.lcp[k]);
                }
                i = phi;
                continue;
            }
            const std::string &v = f.terms[f.sorted[i]];
            size_t d = std::min<size_t>(std::min<size_t>(f.lcp[i], carry), valid);
            carry = 0xffffffffu;
            bool pruned = false;
            while (d < v.size()) {
                d++;
                if (dp.size() <= d) dp.emplace_back(m + 1);
                std::vector<uint32_t> &row = dp[d];
                const std::vector<uint32_t> &pr = dp[d - 1];
                row[0] = (uint32_t)d;
                uint32_t mn = row[0];
                const char ch = v[d - 1];
                for (size_t j = 1; j <= m; j++) {
                    const uint32_t c = std::min(std::min(pr[j] + 1, row[j - 1] + 1), pr[j - 1] + (tok[j - 1] != ch ? 1u : 0u));
                    row[j] = c;
                    mn = std::min(mn, c);
                }
                if (mn > t) { pruned = true; break; }
            }
            valid = d;
            if (pruned) {   // every term sharing v[0..d) is out: hop to the end of that prefix subtree.  (It cannot
                            // hold a prefix match: v[0..d) != tok[0..d), else dp[d][d] = 0 would have kept the row alive.)
                size_t k = i + 1;
                while (k < V && f.lcp[k] >= d) k = f.next_smaller[k];
                i = k;      // lcp[k] < d <= every skipped lcp: the landing position's own lcp is the shared prefix
                continue;
            }
            if (dp[v.size()][m] <= t) emit(f.sorted[i], v.size() == m && v == tok);
            i++;
        }
    }

    std::vector<FieldDict> fields_;
    uint64_t gen_ = 0;
    std::shared_mutex mu_;
    StemFn stem_ = nullptr;
    void *stem_user_ = nullptr;
};

}  // namespace ocd
