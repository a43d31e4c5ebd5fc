// comm.h — NCCL over NVLink for the collectives the path has: an all-gather of per-shard
// top-k records per query batch (SURVEY.md §8e) and, only when corpus df must be counted
// (filters / multi-term tokens / tombstones), an all-reduce of the per-token df counters.  libnccl is bound with
// dlopen/dlsym (no link-time dependency, no header needed): the torch-bundled
// libnccl.so.2 already mapped into a torchrun worker is reused, else the system one.
// A second transport joins several contexts of one process (oc_comm_init_local, e.g. ranks sharing one GPU): the
// same collectives through host memory (comm_local.h), each rank on its own thread.
#pragma once
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <stdint.h>

#include <cstdio>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "comm_local.h"

struct OcComm {
    typedef struct { char internal[128]; } UniqueId;   // ncclUniqueId
    typedef void *Comm;                                // ncclComm_t
    typedef int (*GetUniqueId_t)(UniqueId *);
    typedef int (*CommInitRank_t)(Comm *, int, UniqueId, int);
    typedef int (*AllGather_t)(const void *, void *, size_t, int, Comm, cudaStream_t);
    typedef int (*AllReduce_t)(const void *, void *, size_t, int, int, Comm, cudaStream_t);
    typedef int (*CommDestroy_t)(Comm);
    typedef const char *(*GetErrorString_t)(int);

    Comm comm = nullptr;
    int world = 1, rank = 0;

    struct Api {
        void *h = nullptr;
        GetUniqueId_t GetUniqueId = nullptr;
        CommInitRank_t CommInitRank = nullptr;
        AllGather_t AllGather = nullptr;
        AllReduce_t AllReduce = nullptr;
        CommDestroy_t CommDestroy = nullptr;
        GetErrorString_t GetErrorString = nullptr;
    };
    static Api &api() { static Api a; return a; }

    static bool load(std::string *err) {
        Api &a = api();
        if (a.h) return true;
        const char *names[] = {"libnccl.so.2", "libnccl.so"};
        for (const char *n : names) {
            a.h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
            if (a.h) break;
        }
        if (!a.h) { if (err) *err = std::string("cannot dlopen libnccl.so.2: ") + dlerror(); return false; }
        a.GetUniqueId = (GetUniqueId_t)dlsym(a.h, "ncclGetUniqueId");
        a.CommInitRank = (CommInitRank_t)dlsym(a.h, "ncclCommInitRank");
        a.AllGather = (AllGather_t)dlsym(a.h, "ncclAllGather");
        a.AllReduce = (AllReduce_t)dlsym(a.h, "ncclAllReduce");
        a.CommDestroy = (CommDestroy_t)dlsym(a.h, "ncclCommDestroy");
        a.GetErrorString = (GetErrorString_t)dlsym(a.h, "ncclGetErrorString");
        if (!a.GetUniqueId || !a.CommInitRank || !a.AllGather || !a.AllReduce || !a.CommDestroy) {
            if (err) *err = "libnccl is missing required symbols";
            a.h = nullptr;
            return false;
        }
        return true;
    }
    static std::string estr(int rc) {
        Api &a = api();
        return a.GetErrorString ? std::string(a.GetErrorString(rc)) : std::to_string(rc);
    }
    static bool unique_id(uint8_t out[128], std::string *err) {
        if (!load(err)) return false;
        UniqueId id;
        int rc = api().GetUniqueId(&id);
        if (rc != 0) { if (err) *err = "ncclGetUniqueId: " + estr(rc); return false; }
        memcpy(out, id.internal, 128);
        return true;
    }
    bool init(int world_size, int my_rank, const uint8_t id_bytes[128], std::string *err) {
        if (!load(err)) return false;
        destroy();
        UniqueId id;
        memcpy(id.internal, id_bytes, 128);
        int rc = api().CommInitRank(&comm, world_size, id, my_rank);
        if (rc != 0) { comm = nullptr; if (err) *err = "ncclCommInitRank: " + estr(rc); return false; }
        world = world_size; rank = my_rank;
        return true;
    }
    // in-process group: this rank's view of it and its host staging buffers
    std::shared_ptr<LocalGroup> local;
    std::vector<uint8_t> h_send, h_recv;

    void init_local(std::shared_ptr<LocalGroup> g, int my_rank) {
        destroy();
        local = std::move(g); world = local->world(); rank = my_rank;
    }
    bool ready() const { return comm != nullptr || local != nullptr || world == 1; }
    // bytes per rank; ncclInt8 = 0
    bool all_gather(const void *send, void *recv, size_t bytes, cudaStream_t s, std::string *err) {
        if (local) {
            h_send.resize(bytes); h_recv.resize(bytes * world);
            if (!to_host(h_send.data(), send, bytes, s, err)) return false;
            if (!local->all_gather(rank, h_send.data(), h_recv.data(), bytes, err)) return false;
            return to_device(recv, h_recv.data(), bytes * world, s, err);
        }
        int rc = api().AllGather(send, recv, bytes, /*ncclInt8*/ 0, comm, s);
        if (rc != 0) { if (err) *err = "ncclAllGather: " + estr(rc); return false; }
        return true;
    }
    // in-place-capable sum of `count` uint32 counters; ncclUint32 = 3, ncclSum = 0
    bool all_reduce_sum_u32(const void *send, void *recv, size_t count, cudaStream_t s, std::string *err) {
        if (local) {
            h_send.resize(count * 4); h_recv.resize(count * 4);
            if (!to_host(h_send.data(), send, count * 4, s, err)) return false;
            if (!local->all_reduce_sum_u32(rank, reinterpret_cast<const uint32_t *>(h_send.data()),
                                           reinterpret_cast<uint32_t *>(h_recv.data()), count, err)) return false;
            return to_device(recv, h_recv.data(), count * 4, s, err);
        }
        int rc = api().AllReduce(send, recv, count, /*ncclUint32*/ 3, /*ncclSum*/ 0, comm, s);
        if (rc != 0) { if (err) *err = "ncclAllReduce: " + estr(rc); return false; }
        return true;
    }
    void destroy() {
        if (comm) api().CommDestroy(comm);
        if (local) local->leave(rank);
        comm = nullptr; local.reset(); world = 1; rank = 0;
    }

private:
    // the local transport's staging: the rank's stream is drained first, so its own device work never waits on a peer
    static bool to_host(void *dst, const void *src, size_t bytes, cudaStream_t s, std::string *err) {
        cudaError_t e = cudaStreamSynchronize(s);
        if (e == cudaSuccess && bytes) e = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        if (e != cudaSuccess && err) *err = std::string("local group staging: ") + cudaGetErrorString(e);
        return e == cudaSuccess;
    }
    static bool to_device(void *dst, const void *src, size_t bytes, cudaStream_t s, std::string *err) {
        cudaError_t e = bytes ? cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, s) : cudaSuccess;
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        if (e != cudaSuccess && err) *err = std::string("local group staging: ") + cudaGetErrorString(e);
        return e == cudaSuccess;
    }
};
