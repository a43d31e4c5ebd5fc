// dense_cache.h — the dense contribution arrays of hot BM25 terms, kept on the device across search calls.
//
// A hot term's array (float[n_tiles * BM25_TILE], the contribution c of each posting scattered to its row, 0 elsewhere;
// bm25_precompute_kernel, followed in the same allocation by its summary, a presence bitmap and per-tile bounds that
// the same kernel sets: bm25_dense_bytes) depends only on the string snapshot's postings, the term's field weight and idf, bm25_k
// and bm25_b (the derived postings), and the row bitmap.  Calls without a row bitmap (no filter, no tombstones, no df
// counted on the device) key the array by those values and reuse it: the same kernel wrote it with the same rounded
// ops, so a later call reads the bits it would have built.  DESIGN.md §4 "Dense-array cache".
//
// Ordering: calls on a ctx serialise on its lock.  An array is built (memset + precompute) on the stream the call's
// fulltext stage uses and read on that stream and, after the side stream is joined into it, on the main stream.  A
// call's side stream first waits on the call's EV_H2D, recorded on the main stream after every earlier call's work, so
// a later call's reads, and the stream-ordered free (cudaFreeAsync) of an evicted array whose memory a later
// cudaMallocAsync may hand out again, come after every earlier write and read of it.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <memory>
#include <unordered_map>

struct StrSnap;

struct DenseKey {
    uint64_t snap;                  // StrSnap::ident: changes on every commit, load and in-place change of the snapshot
    uint64_t term;                  // field << 32 | term id
    uint32_t weight, idf, k, b;     // float bits
    bool operator==(const DenseKey &o) const {
        return snap == o.snap && term == o.term && weight == o.weight && idf == o.idf && k == o.k && b == o.b;
    }
};
struct DenseKeyHash {
    size_t operator()(const DenseKey &x) const {
        uint64_t h = x.snap * 0x9E3779B97F4A7C15ull ^ x.term * 0xC2B2AE3D27D4EB4Full;
        h ^= (uint64_t(x.weight) << 32 | x.idf) * 0x165667B19E3779F9ull;
        h ^= (uint64_t(x.k) << 32 | x.b) * 0x27D4EB2F165667C5ull;
        return size_t(h ^ (h >> 29));
    }
};
struct DenseEntry {
    float *p = nullptr;             // cudaMallocAsync'd
    uint64_t bytes = 0;
    uint64_t last_use = 0;          // DenseCache::tick of the last call that read it
    bool ready = false;             // its build was enqueued (a call that failed before that leaves it false)
    std::weak_ptr<StrSnap> snap;    // dropped once the snapshot is gone or its ident moved on
};
struct DenseCache {
    using Map = std::unordered_map<DenseKey, DenseEntry, DenseKeyHash>;
    Map map;
    uint64_t used = 0;              // bytes held
    uint64_t in_call = 0;           // bytes the current call reads (not evictable)
    uint64_t tick = 0;              // calls that looked the cache up
    Map::iterator drop(Map::iterator it, cudaStream_t st) {
        cudaFreeAsync(it->second.p, st);
        used -= it->second.bytes;
        return map.erase(it);
    }
    // the least recently used array the current call does not read; false when there is none
    bool evict_one(cudaStream_t st) {
        auto lru = map.end();
        for (auto it = map.begin(); it != map.end(); ++it)
            if (it->second.last_use != tick && (lru == map.end() || it->second.last_use < lru->second.last_use)) lru = it;
        if (lru == map.end()) return false;
        drop(lru, st);
        return true;
    }
    void clear(cudaStream_t st) {
        for (auto it = map.begin(); it != map.end();) it = drop(it, st);
    }
};
