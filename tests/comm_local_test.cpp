// Host test of the in-process collective group (oramacore_b200/csrc/comm_local.h): W threads, one per rank, run many
// rounds of gathers and sums whose results are checked against a plain loop over what every rank sent.  Scenarios
// (one per process): rounds W | mismatch | leave | timeout.  Built and run by tests/test_comm_local_host.py (g++, no
// CUDA), at -O2 and under ThreadSanitizer.  Prints "wrong=0" when every check held.
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "../oramacore_b200/csrc/comm_local.h"

static std::atomic<long> g_wrong{0}, g_checked{0};
#define CHECK(c, ...)                                          \
    do {                                                       \
        g_checked++;                                           \
        if (!(c)) {                                            \
            if (g_wrong++ < 20) { fprintf(stderr, __VA_ARGS__); fputc('\n', stderr); } \
        }                                                      \
    } while (0)

// what rank r sends in round i: bytes and counters derived from (round, rank, position) only
static uint8_t byte_of(int i, int r, size_t j) { return uint8_t(i * 131 + r * 31 + j * 7 + (j >> 8)); }
static uint32_t word_of(int i, int r, size_t j) { return uint32_t(i) * 2654435761u + uint32_t(r) * 40503u + uint32_t(j) * 97u + 0xfffffff0u * (r & 1); }
static size_t gather_bytes(int i) { return i % 7 == 0 ? 0 : size_t((i * 37) % 1500); }   // 0-byte gathers every 7th round
static size_t sum_count(int i) { return i % 11 == 0 ? 0 : size_t((i * 53) % 700); }

static void rounds(int W, int n_rounds) {
    LocalGroup g(W);
    std::vector<std::thread> th;
    for (int r = 0; r < W; r++)
        th.emplace_back([&, r] {
            std::vector<uint8_t> send, recv;
            std::vector<uint32_t> ws, wr;
            for (int i = 0; i < n_rounds; i++) {
                std::string err;
                if (i % 2 == 0) {
                    const size_t b = gather_bytes(i);
                    send.resize(b);
                    for (size_t j = 0; j < b; j++) send[j] = byte_of(i, r, j);
                    recv.assign(size_t(W) * b + 1, 0xab);   // one guard byte past the result
                    const bool ok = g.all_gather(r, send.data(), recv.data(), b, &err);
                    CHECK(ok, "W=%d rank %d round %d gather failed: %s", W, r, i, err.c_str());
                    bool eq = recv[size_t(W) * b] == 0xab;
                    for (int s = 0; s < W && eq; s++)
                        for (size_t j = 0; j < b; j++)
                            if (recv[size_t(s) * b + j] != byte_of(i, s, j)) { eq = false; break; }
                    CHECK(eq, "W=%d rank %d round %d: wrong gather result (%zu B per rank)", W, r, i, b);
                } else {
                    const size_t n = sum_count(i);
                    ws.resize(n + 1);
                    for (size_t j = 0; j < n; j++) ws[j] = word_of(i, r, j);
                    ws[n] = 0x5a5a5a5au;
                    const bool in_place = i % 3 == 0;   // send == recv, as the df all-reduce calls it
                    wr.assign(n + 1, 0x5a5a5a5au);
                    uint32_t *out = in_place ? ws.data() : wr.data();
                    const bool ok = g.all_reduce_sum_u32(r, ws.data(), out, n, &err);
                    CHECK(ok, "W=%d rank %d round %d sum failed: %s", W, r, i, err.c_str());
                    bool eq = out[n] == 0x5a5a5a5au;
                    for (size_t j = 0; j < n && eq; j++) {
                        uint32_t want = 0;
                        for (int s = 0; s < W; s++) want += word_of(i, s, j);
                        eq = out[j] == want;
                    }
                    CHECK(eq, "W=%d rank %d round %d: wrong sum (%zu counters)", W, r, i, n);
                }
            }
        });
    for (auto &t : th) t.join();
}

// rank-divergent calls: every rank fails, and the next round (all agree) succeeds
static void mismatch(int W) {
    LocalGroup g(W);
    std::vector<std::thread> th;
    std::atomic<int> failed{0};
    for (int r = 0; r < W; r++)
        th.emplace_back([&, r] {
            uint8_t send[64] = {}, recv[64 * 16] = {};
            uint32_t ws[16] = {}, wr[16] = {};
            for (int i = 0; i < 200; i++) {
                std::string err;
                const int kind = i % 4;   // 0: agree, 1: one rank sends a different size, 2: one rank sums, 3: agree
                const int odd = (i / 4) % W;
                bool ok;
                if (kind == 2 && r == odd) ok = g.all_reduce_sum_u32(r, ws, wr, 4, &err);
                else ok = g.all_gather(r, send, recv, (kind == 1 && r == odd) ? 8 : 16, &err);
                const bool expect = kind == 0 || kind == 3;
                CHECK(ok == expect, "W=%d rank %d round %d kind %d: ok=%d (%s)", W, r, i, kind, ok, err.c_str());
                if (!ok) {
                    failed++;
                    CHECK(err.find("different collectives") != std::string::npos, "rank %d: unexpected message %s", r, err.c_str());
                }
            }
        });
    for (auto &t : th) t.join();
    CHECK(failed == W * 100, "W=%d: %d failures, expected %d", W, failed.load(), W * 100);
}

// a rank leaves (its context is shut down) while the others wait in a round, then they call again: every call fails
// at once, well before the timeout
static void leave(int W) {
    LocalGroup g(W, std::chrono::seconds(30));
    const auto t0 = std::chrono::steady_clock::now();
    std::vector<std::thread> th;
    for (int r = 0; r < W; r++)
        th.emplace_back([&, r] {
            uint32_t w[4] = {1, 2, 3, 4};
            std::string err;
            CHECK(g.all_reduce_sum_u32(r, w, w, 4, &err), "rank %d: first round failed: %s", r, err.c_str());
            CHECK(w[0] == uint32_t(W), "rank %d: first round sum %u", r, w[0]);
            if (r == W - 1) {
                std::this_thread::sleep_for(std::chrono::milliseconds(50));   // the others are waiting by now
                g.leave(r);
                return;
            }
            for (int k = 0; k < 2; k++) {
                const bool ok = g.all_reduce_sum_u32(r, w, w, 4, &err);
                CHECK(!ok && err.find("left the group") != std::string::npos, "rank %d call %d after leave: ok=%d (%s)", r, k, ok, err.c_str());
            }
        });
    for (auto &t : th) t.join();
    const double s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    CHECK(s < 10.0, "W=%d: leave took %.1f s to fail the waiting ranks", W, s);
}

// rank W-1 never arrives: the others fail after the timeout with its number in the message, and the group is broken
static void timeout(int W) {
    LocalGroup g(W, std::chrono::milliseconds(200));
    std::atomic<int> waited{0};   // ranks that waited out the timeout (a rank arriving after it fails at once)
    std::vector<std::thread> th;
    for (int r = 0; r + 1 < W; r++)
        th.emplace_back([&, r] {
            uint8_t b[8] = {};
            std::vector<uint8_t> out(8 * size_t(W));
            std::string err;
            const auto t0 = std::chrono::steady_clock::now();
            const bool ok = g.all_gather(r, b, out.data(), 8, &err);
            const double s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
            // the missing ranks are listed in ascending order, so the absent one ends the list
            const std::string tail = " " + std::to_string(W - 1);
            CHECK(!ok && err.find("timed out after 200 ms") != std::string::npos, "rank %d: ok=%d (%s)", r, ok, err.c_str());
            CHECK(err.size() > tail.size() && err.compare(err.size() - tail.size(), tail.size(), tail) == 0,
                  "rank %d: the missing rank is not named: %s", r, err.c_str());
            CHECK(s < 10.0, "rank %d: failed after %.3f s", r, s);
            if (s >= 0.15) waited++;
            CHECK(!g.all_gather(r, b, out.data(), 8, &err), "rank %d: a broken group succeeded", r);
        });
    for (auto &t : th) t.join();
    CHECK(waited > 0, "W=%d: no rank waited for the timeout", W);
    std::string err;
    uint8_t b[8] = {};
    std::vector<uint8_t> out(8 * size_t(W));
    CHECK(!g.all_gather(W - 1, b, out.data(), 8, &err), "the late rank succeeded in a broken group");
}

int main(int argc, char **argv) {
    const std::string sc = argc > 1 ? argv[1] : "";
    if (sc == "rounds" && argc > 2) {
        const int W = atoi(argv[2]);
        rounds(W, W >= 16 ? 2000 : 5000);
    } else if (sc == "mismatch") {
        for (int W : {2, 3, 16}) mismatch(W);
    } else if (sc == "leave") {
        for (int W : {2, 3, 16}) leave(W);
    } else if (sc == "timeout") {
        for (int W : {2, 3, 16}) timeout(W);
    } else {
        fprintf(stderr, "usage: comm_local_test rounds W | mismatch | leave | timeout\n");
        return 2;
    }
    printf("checked=%ld wrong=%ld\n", g_checked.load(), g_wrong.load());
    return g_wrong ? 1 : 0;
}
