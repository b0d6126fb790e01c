// C entry points over the session table of the live-stream sets (fluidaudio_b200/csrc/session_table.h, compiled with
// this file by g++), for tests/test_session_table.py.  The table's Session is a two-field probe; the grow and init
// callbacks return the status the caller asks for and record what they were called with.
#include "session_table.h"

#include <cstdarg>
#include <cstdio>

namespace fa {
static char g_error[512] = "";
void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_error, sizeof(g_error), fmt, ap);
    va_end(ap);
}
const char *last_error() { return g_error; }
} // namespace fa

struct Probe {
    long long value;
    int tag;
};
using Table = fa::SessionTable<Probe>;

extern "C" {

void *st_create() { return new Table(); }
void st_destroy(void *t) { delete static_cast<Table *>(t); }
const char *st_last_error() { return fa::last_error(); }
int st_slots(const void *t) { return static_cast<const Table *>(t)->slots(); }
int st_valid(const void *t, int id) { return static_cast<const Table *>(t)->valid(id); }

// grown_to: the slot count grow was called with, or -1; init_id: the id init was called with, or -1
int st_open(void *t, int min_slots, int grow_status, int init_status, int *id, int *grown_to, int *init_id) {
    *grown_to = *init_id = -1;
    auto grow = [&](int slots) {
        *grown_to = slots;
        return grow_status;
    };
    auto init = [&](int i) {
        *init_id = i;
        return init_status;
    };
    return static_cast<Table *>(t)->open(min_slots, grow, init, id);
}

int st_close(void *t, int id, const char *where) { return static_cast<Table *>(t)->close(id, where); }
int st_check(const void *t, int count, const int *ids, const char *where) {
    return static_cast<const Table *>(t)->check(count, ids, where);
}

void st_get(const void *t, int id, long long *value, int *tag) {
    const Probe &p = (*static_cast<const Table *>(t))[id];
    *value = p.value;
    *tag = p.tag;
}
void st_set(void *t, int id, long long value, int tag) { (*static_cast<Table *>(t))[id] = Probe{value, tag}; }

void st_commit(void *t, int count, const int *ids, const long long *values, const int *tags) {
    std::vector<Probe> next(count);
    for (int i = 0; i < count; ++i) next[i] = Probe{values[i], tags[i]};
    static_cast<Table *>(t)->commit(count, ids, next.data());
}

} // extern "C"
