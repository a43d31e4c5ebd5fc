// comm_local.h — an in-process collective group: `world` ranks that live in one process (e.g. several contexts
// sharing one GPU, which NCCL refuses) exchange host buffers on the host.  No CUDA here: comm.h stages the device
// buffers through host memory around these calls, so the bytes exchanged are the ones ncclAllGather /
// ncclAllReduce would move.
//
// Each collective is one round: every rank deposits its contribution, the last one to arrive checks that all ranks
// called the same collective (kind and byte count) and builds the result, then every rank copies the result out and
// the next round may begin.  Ranks wait for each other on a condition variable only, with a fixed timeout:
//   - a kind or size mismatch fails the round on every rank (the group stays usable for the next round);
//   - a timeout names the ranks that never arrived and breaks the group (the ranks are out of step: every later
//     collective fails at once);
//   - leave(rank) (its context is shut down) breaks the group as well: pending and later collectives fail at once.
#pragma once
#include <stdint.h>

#include <chrono>
#include <condition_variable>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

class LocalGroup {
public:
    enum Kind : uint32_t { KIND_GATHER = 1, KIND_SUM_U32 = 2 };

    explicit LocalGroup(int world, std::chrono::milliseconds timeout = std::chrono::seconds(60))
        : world_(world), timeout_(timeout), in_(size_t(world)), kind_(size_t(world)), bytes_(size_t(world)),
          present_(size_t(world), 0) {}
    int world() const { return world_; }

    // recv[r * bytes, (r + 1) * bytes) = rank r's send, on every rank; bytes may be 0
    bool all_gather(int rank, const void *send, void *recv, size_t bytes, std::string *err) {
        return round(rank, KIND_GATHER, send, bytes, recv, size_t(world_) * bytes, err);
    }
    // recv[i] = sum over the ranks of send[i] (mod 2^32); send may equal recv
    bool all_reduce_sum_u32(int rank, const uint32_t *send, uint32_t *recv, size_t count, std::string *err) {
        return round(rank, KIND_SUM_U32, send, count * 4, recv, count * 4, err);
    }
    // the rank's context is going away: every rank waiting in a round, and every later collective, fails
    void leave(int rank) {
        std::lock_guard<std::mutex> g(mu_);
        if (broken_.empty()) broken_ = "rank " + std::to_string(rank) + " left the group";
        cv_.notify_all();
    }

private:
    static const char *kind_name(uint32_t k) { return k == KIND_GATHER ? "all_gather" : "all_reduce_sum_u32"; }

    bool round(int rank, uint32_t kind, const void *send, size_t bytes, void *recv, size_t out_bytes, std::string *err) {
        std::unique_lock<std::mutex> lk(mu_);
        const auto deadline = std::chrono::steady_clock::now() + timeout_;
        // the previous round must have been copied out by every rank before its result is replaced
        while (broken_.empty() && departing_)
            if (cv_.wait_until(lk, deadline) == std::cv_status::timeout && departing_) return fail_timeout(err, "to leave the last round");
        if (!broken_.empty()) return set(err, "local group: " + broken_);
        const uint64_t my_round = round_;
        in_[rank].assign(static_cast<const uint8_t *>(send), static_cast<const uint8_t *>(send) + bytes);
        kind_[rank] = kind; bytes_[rank] = bytes; present_[rank] = 1;
        if (++arrived_ == world_) {
            finish();
            cv_.notify_all();
        } else {
            while (broken_.empty() && !(departing_ && round_ == my_round))
                if (cv_.wait_until(lk, deadline) == std::cv_status::timeout && !(departing_ && round_ == my_round)) {
                    fail_timeout(err, "in " + std::string(kind_name(kind)));
                    present_[rank] = 0; arrived_--;
                    return false;
                }
            if (!(departing_ && round_ == my_round)) {   // broken while waiting: withdraw
                present_[rank] = 0; arrived_--;
                return set(err, "local group: " + broken_);
            }
        }
        const bool ok = ok_;
        if (ok && out_bytes) memcpy(recv, out_.data(), out_bytes);
        if (!ok) set(err, msg_);
        if (++departed_ == world_) {   // the last one out opens the next round
            departing_ = false; departed_ = 0; arrived_ = 0; round_++;
            for (auto &v : present_) v = 0;
            cv_.notify_all();
        }
        return ok;
    }

    // every rank has arrived: check that they agree, then gather or sum
    void finish() {
        ok_ = true; msg_.clear();
        for (int r = 1; r < world_; r++)
            if (kind_[r] != kind_[0] || bytes_[r] != bytes_[0]) ok_ = false;
        if (!ok_) {
            msg_ = "local group: the ranks called different collectives:";
            for (int r = 0; r < world_; r++)
                msg_ += " rank " + std::to_string(r) + " " + kind_name(kind_[r]) + "(" + std::to_string(bytes_[r]) + " B)";
        } else if (kind_[0] == KIND_GATHER) {
            const size_t b = bytes_[0];
            out_.resize(size_t(world_) * b);
            for (int r = 0; r < world_; r++) if (b) memcpy(out_.data() + size_t(r) * b, in_[r].data(), b);
        } else {
            const size_t n = bytes_[0] / 4;
            out_.assign(bytes_[0], 0);
            uint32_t *o = reinterpret_cast<uint32_t *>(out_.data());
            for (int r = 0; r < world_; r++) {
                const uint8_t *src = in_[r].data();
                for (size_t i = 0; i < n; i++) { uint32_t v; memcpy(&v, src + 4 * i, 4); o[i] += v; }
            }
        }
        departing_ = true;
    }

    bool fail_timeout(std::string *err, const std::string &where) {
        std::string missing;
        for (int r = 0; r < world_; r++)
            if (!present_[r]) missing += (missing.empty() ? "" : ", ") + std::to_string(r);
        const std::string m = "timed out after " + std::to_string(timeout_.count()) + " ms " + where +
                              (departing_ ? "" : " waiting for rank(s) " + missing);
        if (broken_.empty()) broken_ = m;
        cv_.notify_all();
        return set(err, "local group: " + m);
    }
    static bool set(std::string *err, const std::string &m) {
        if (err) *err = m;
        return false;
    }

    const int world_;
    const std::chrono::milliseconds timeout_;
    std::mutex mu_;
    std::condition_variable cv_;
    std::vector<std::vector<uint8_t>> in_;   // [rank] contribution of the current round
    std::vector<uint32_t> kind_;
    std::vector<size_t> bytes_;
    std::vector<uint8_t> present_;           // [rank] arrived in the current round
    std::vector<uint8_t> out_;               // the round's result
    int arrived_ = 0, departed_ = 0;
    bool departing_ = false, ok_ = true;
    uint64_t round_ = 0;
    std::string msg_, broken_;
};
