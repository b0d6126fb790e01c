// The open ids of a live-stream set (mel_stream.cu, sortformer_streams.cu), a host mirror per slot and the slot count
// the set's per-session device arrays are sized for.  A push checks its ids and plans every session's next mirror
// before anything runs, then commits the plan once its device work succeeded: a failed push changes no session.
// Plain C++ (no CUDA), so the CPU test-suite compiles it with g++ (tests/emul/session_table_shim.cpp).
#pragma once

#include "fa_common.cuh"

#include <algorithm>
#include <cstdint>
#include <vector>

namespace fa {

template <typename Session> class SessionTable {
  public:
    int slots() const { return (int)live_.size(); }
    bool valid(int id) const { return id >= 0 && id < slots() && live_[id]; }
    Session &operator[](int id) { return mirror_[id]; }
    const Session &operator[](int id) const { return mirror_[id]; }

    // Opens the lowest closed id (ids are dense from 0) with a value-initialised mirror, which init(id) completes along
    // with the session's device state.  A full table first calls grow(max(min_slots, 2 * slots)) to resize the caller's
    // arrays.  If either fails, open returns its status and the id stays closed; a failed grow changes nothing.
    template <typename Grow, typename Init> int open(int min_slots, Grow &&grow, Init &&init, int *id) {
        int i = 0;
        while (i < slots() && live_[i]) ++i;
        if (i == slots()) {
            const int grown = std::max(min_slots, 2 * slots());
            const int st = grow(grown);
            if (st != FA_OK) return st;
            live_.resize(grown, 0);
            mirror_.resize(grown);
        }
        mirror_[i] = Session{};
        const int st = init(i);
        if (st != FA_OK) return st;
        live_[i] = 1;
        *id = i;
        return FA_OK;
    }

    int close(int id, const char *where) {
        const int st = check(1, &id, where);
        if (st == FA_OK) live_[id] = 0;
        return st;
    }

    // Every id is open and none appears twice, or FA_INVALID_ARGUMENT with the error text under the prefix `where`.
    int check(int count, const int *ids, const char *where) const {
        std::vector<uint8_t> seen(slots(), 0);
        for (int i = 0; i < count; ++i) {
            const int id = ids[i];
            if (!valid(id)) {
                set_error("%s: session %d is not open", where, id);
                return FA_INVALID_ARGUMENT;
            }
            if (seen[id]) {
                set_error("%s: session %d appears twice", where, id);
                return FA_INVALID_ARGUMENT;
            }
            seen[id] = 1;
        }
        return FA_OK;
    }

    // Session ids[i] becomes next[i].
    void commit(int count, const int *ids, const Session *next) {
        for (int i = 0; i < count; ++i) mirror_[ids[i]] = next[i];
    }

  private:
    std::vector<uint8_t> live_;
    std::vector<Session> mirror_;
};

} // namespace fa
