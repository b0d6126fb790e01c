// Embedding-export files: the on-disk input format of the clustering backend (SURVEY.md 8f rank 2).
//
// The reference writes them from OfflineDiarizerManager.exportEmbeddings (OfflineDiarizerManager.swift:913-955,
// enabled by OfflineDiarizerConfig.embeddingExportPath): one JSON array of objects
//   {chunkIndex, speakerIndex, startFrame, endFrame, startTime, endTime, embedding256:[Float], rho128:[Double], cluster}
// produced by Foundation's JSONEncoder (keys in any order, numbers in shortest round-trip form, optional exponent).
// Reading such a dump gives the backend real FluidAudio inputs (and the labels the reference assigned) without CoreML.
//
// Host code only (no kernels): a small recursive-descent reader for exactly this schema.  Numbers are converted with
// strtof / strtod straight from the decimal text, so a float32 written in shortest form reads back bit-identically.
#include "c_abi.h"

#include <cerrno>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

namespace {

struct Reader {
    const char *p, *end;
    std::string err;

    void ws() {
        while (p < end && (*p == ' ' || *p == '\n' || *p == '\t' || *p == '\r')) ++p;
    }
    bool fail(const char *what) {
        if (err.empty()) {
            char buf[160];
            std::snprintf(buf, sizeof buf, "%s at byte %lld", what, (long long)(p - start));
            err = buf;
        }
        return false;
    }
    bool expect(char c) {
        ws();
        if (p >= end || *p != c) return fail(c == '[' ? "expected '['" : c == '{' ? "expected '{'" : c == ':' ? "expected ':'" : "unexpected character");
        ++p;
        return true;
    }
    bool peek(char c) {
        ws();
        return p < end && *p == c;
    }
    // keys of this schema contain no escapes; values of unknown keys are skipped structurally
    bool key(std::string &out) {
        ws();
        if (p >= end || *p != '"') return fail("expected a key");
        const char *q = ++p;
        while (p < end && *p != '"') {
            if (*p == '\\') ++p;
            ++p;
        }
        if (p >= end) return fail("unterminated string");
        out.assign(q, p - q);
        ++p;
        return true;
    }
    bool number_token(const char *&tok_end) {
        ws();
        const char *q = p;
        if (q < end && (*q == '-' || *q == '+')) ++q;
        bool digits = false;
        while (q < end && ((*q >= '0' && *q <= '9') || *q == '.' || *q == 'e' || *q == 'E' || *q == '-' || *q == '+')) {
            if (*q >= '0' && *q <= '9') digits = true;
            ++q;
        }
        if (!digits) return fail("expected a number");
        tok_end = q;
        return true;
    }
    bool f64(double &v) {
        const char *te;
        if (!number_token(te)) return false;
        char tmp[64];
        const size_t n = (size_t)(te - p);
        if (n >= sizeof tmp) return fail("number too long");
        std::memcpy(tmp, p, n);
        tmp[n] = 0;
        char *e2 = nullptr;
        v = std::strtod(tmp, &e2);
        if (e2 != tmp + n) return fail("malformed number");
        p = te;
        return true;
    }
    bool f32(float &v) {
        const char *te;
        if (!number_token(te)) return false;
        char tmp[64];
        const size_t n = (size_t)(te - p);
        if (n >= sizeof tmp) return fail("number too long");
        std::memcpy(tmp, p, n);
        tmp[n] = 0;
        char *e2 = nullptr;
        v = std::strtof(tmp, &e2);
        if (e2 != tmp + n) return fail("malformed number");
        p = te;
        return true;
    }
    bool i64(long long &v) {
        double d;
        if (!f64(d)) return false;
        if (d != std::floor(d) || std::fabs(d) > 9.0e15) return fail("expected an integer");
        v = (long long)d;
        return true;
    }
    bool skip_value() {
        struct Depth {
            int &d;
            explicit Depth(int &x) : d(x) { ++d; }
            ~Depth() { --d; }
        } guard(depth);
        if (depth > 64) return fail("values nested deeper than 64 levels");
        ws();
        if (p >= end) return fail("unexpected end");
        if (*p == '"') {
            std::string s;
            return key(s);
        }
        if (*p == '[' || *p == '{') {
            const char open = *p, close = open == '[' ? ']' : '}';
            ++p;
            if (peek(close)) {
                ++p;
                return true;
            }
            for (;;) {
                if (open == '{') {
                    std::string k;
                    if (!key(k) || !expect(':')) return false;
                }
                if (!skip_value()) return false;
                ws();
                if (p < end && *p == ',') {
                    ++p;
                    continue;
                }
                if (p < end && *p == close) {
                    ++p;
                    return true;
                }
                return fail("expected ',' or a closing bracket");
            }
        }
        if (end - p >= 4 && (!std::memcmp(p, "true", 4) || !std::memcmp(p, "null", 4))) {
            p += 4;
            return true;
        }
        if (end - p >= 5 && !std::memcmp(p, "false", 5)) {
            p += 5;
            return true;
        }
        double d;
        return f64(d);
    }
    const char *start;
    int depth = 0;   // nesting of skipped values: bounded so that a file of '[[[[...' cannot exhaust the stack
};

struct Entry {
    long long chunk = 0, speaker = 0, start_frame = 0, end_frame = 0, cluster = -1;
    double start_time = 0, end_time = 0;
    std::vector<float> emb;
    std::vector<double> rho;
};

template <typename T, typename F> bool read_array(Reader &r, std::vector<T> &out, F one) {
    out.clear();
    if (!r.expect('[')) return false;
    if (r.peek(']')) {
        ++r.p;
        return true;
    }
    for (;;) {
        T v;
        if (!one(v)) return false;
        out.push_back(v);
        r.ws();
        if (r.p < r.end && *r.p == ',') {
            ++r.p;
            continue;
        }
        if (r.p < r.end && *r.p == ']') {
            ++r.p;
            return true;
        }
        return r.fail("expected ',' or ']'");
    }
}

bool read_entry(Reader &r, Entry &e) {
    if (!r.expect('{')) return false;
    if (r.peek('}')) {
        ++r.p;
        return true;
    }
    for (;;) {
        std::string k;
        if (!r.key(k) || !r.expect(':')) return false;
        bool ok;
        if (k == "chunkIndex") ok = r.i64(e.chunk);
        else if (k == "speakerIndex") ok = r.i64(e.speaker);
        else if (k == "startFrame") ok = r.i64(e.start_frame);
        else if (k == "endFrame") ok = r.i64(e.end_frame);
        else if (k == "cluster") ok = r.i64(e.cluster);
        else if (k == "startTime") ok = r.f64(e.start_time);
        else if (k == "endTime") ok = r.f64(e.end_time);
        else if (k == "embedding256") ok = read_array(r, e.emb, [&](float &v) { return r.f32(v); });
        else if (k == "rho128") ok = read_array(r, e.rho, [&](double &v) { return r.f64(v); });
        else ok = r.skip_value();
        if (!ok) return false;
        r.ws();
        if (r.p < r.end && *r.p == ',') {
            ++r.p;
            continue;
        }
        if (r.p < r.end && *r.p == '}') {
            ++r.p;
            return true;
        }
        return r.fail("expected ',' or '}'");
    }
}

int load_file(const char *path, std::vector<char> &buf) {
    FILE *f = std::fopen(path, "rb");
    if (!f) {
        fa::set_error("cannot open %s: %s", path, std::strerror(errno));
        return FA_INVALID_ARGUMENT;
    }
    std::fseek(f, 0, SEEK_END);
    const long sz = std::ftell(f);
    std::fseek(f, 0, SEEK_SET);
    buf.resize(sz > 0 ? (size_t)sz : 0);
    const size_t got = buf.empty() ? 0 : std::fread(buf.data(), 1, buf.size(), f);
    std::fclose(f);
    if (got != buf.size()) {
        fa::set_error("short read on %s", path);
        return FA_RUNTIME_ERROR;
    }
    return FA_OK;
}

int parse(const char *path, std::vector<Entry> &entries) {
    std::vector<char> buf;
    const int st = load_file(path, buf);
    if (st != FA_OK) return st;
    Reader r{buf.data(), buf.data() + buf.size(), {}, buf.data()};
    entries.clear();
    bool ok = r.expect('[');
    if (ok && r.peek(']')) {
        ++r.p;
    } else if (ok) {
        for (;;) {
            entries.emplace_back();
            if (!(ok = read_entry(r, entries.back()))) break;
            r.ws();
            if (r.p < r.end && *r.p == ',') {
                ++r.p;
                continue;
            }
            if (r.p < r.end && *r.p == ']') {
                ++r.p;
                break;
            }
            ok = r.fail("expected ',' or ']'");
            break;
        }
    }
    if (ok) {
        r.ws();
        if (r.p != r.end) ok = r.fail("trailing characters");
    }
    if (!ok) {
        fa::set_error("%s: %s", path, r.err.c_str());
        return FA_INVALID_ARGUMENT;
    }
    return FA_OK;
}

} // namespace

FA_API fa_status fa_export_shape(const char *path, size_t *count, size_t *emb_dim, size_t *rho_dim) {
    return fa::guard(__func__, [&]() -> int {
        if (!path || !count || !emb_dim || !rho_dim) return FA_INVALID_ARGUMENT;
        std::vector<Entry> entries;
        const int st = parse(path, entries);
        if (st != FA_OK) return st;
        *count = entries.size();
        *emb_dim = entries.empty() ? 0 : entries[0].emb.size();
        *rho_dim = entries.empty() ? 0 : entries[0].rho.size();
        for (const Entry &e : entries)
            if (e.emb.size() != *emb_dim || e.rho.size() != *rho_dim) {
                fa::set_error("%s: entries have different embedding256 / rho128 lengths", path);
                return FA_INVALID_ARGUMENT;
            }
        return FA_OK;
    });
}

FA_API fa_status fa_export_read(const char *path, size_t count, size_t emb_dim, size_t rho_dim, int32_t *chunk_index,
                         int32_t *speaker_index, int32_t *start_frame, int32_t *end_frame, double *start_time,
                         double *end_time, float *emb, double *rho, int32_t *cluster) {
    return fa::guard(__func__, [&]() -> int {
        if (!path) return FA_INVALID_ARGUMENT;
        std::vector<Entry> entries;
        const int st = parse(path, entries);
        if (st != FA_OK) return st;
        if (entries.size() != count) {
            fa::set_error("%s holds %zu entries, caller expected %zu", path, entries.size(), count);
            return FA_INVALID_ARGUMENT;
        }
        for (size_t i = 0; i < count; ++i) {
            const Entry &e = entries[i];
            if (e.emb.size() != emb_dim || e.rho.size() != rho_dim) {
                fa::set_error("%s: entry %zu has %zu / %zu values, expected %zu / %zu", path, i, e.emb.size(), e.rho.size(),
                              emb_dim, rho_dim);
                return FA_INVALID_ARGUMENT;
            }
            if (chunk_index) chunk_index[i] = (int32_t)e.chunk;
            if (speaker_index) speaker_index[i] = (int32_t)e.speaker;
            if (start_frame) start_frame[i] = (int32_t)e.start_frame;
            if (end_frame) end_frame[i] = (int32_t)e.end_frame;
            if (start_time) start_time[i] = e.start_time;
            if (end_time) end_time[i] = e.end_time;
            if (cluster) cluster[i] = (int32_t)e.cluster;
            if (emb) std::memcpy(emb + i * emb_dim, e.emb.data(), sizeof(float) * emb_dim);
            if (rho) std::memcpy(rho + i * rho_dim, e.rho.data(), sizeof(double) * rho_dim);
        }
        return FA_OK;
    });
}

FA_API fa_status fa_export_write(const char *path, size_t count, size_t emb_dim, size_t rho_dim, const int32_t *chunk_index,
                          const int32_t *speaker_index, const int32_t *start_frame, const int32_t *end_frame,
                          const double *start_time, const double *end_time, const float *emb, const double *rho,
                          const int32_t *cluster) {
    return fa::guard(__func__, [&]() -> int {
        if (!path || (count && (!emb || !rho))) return FA_INVALID_ARGUMENT;
        FILE *f = std::fopen(path, "wb");
        if (!f) {
            fa::set_error("cannot create %s: %s", path, std::strerror(errno));
            return FA_INVALID_ARGUMENT;
        }
        std::fputc('[', f);
        for (size_t i = 0; i < count; ++i) {
            if (i) std::fputc(',', f);
            std::fprintf(f, "{\"chunkIndex\":%d,\"speakerIndex\":%d,\"startFrame\":%d,\"endFrame\":%d,",
                         chunk_index ? chunk_index[i] : 0, speaker_index ? speaker_index[i] : 0,
                         start_frame ? start_frame[i] : 0, end_frame ? end_frame[i] : 0);
            std::fprintf(f, "\"startTime\":%.17g,\"endTime\":%.17g,\"embedding256\":[", start_time ? start_time[i] : 0.0,
                         end_time ? end_time[i] : 0.0);
            for (size_t k = 0; k < emb_dim; ++k) std::fprintf(f, k ? ",%.9g" : "%.9g", (double)emb[i * emb_dim + k]);
            std::fputs("],\"rho128\":[", f);
            for (size_t k = 0; k < rho_dim; ++k) std::fprintf(f, k ? ",%.17g" : "%.17g", rho[i * rho_dim + k]);
            std::fprintf(f, "],\"cluster\":%d}", cluster ? cluster[i] : -1);
        }
        std::fputc(']', f);
        const bool bad = std::ferror(f) != 0;
        if (std::fclose(f) != 0 || bad) {
            fa::set_error("write error on %s", path);
            return FA_RUNTIME_ERROR;
        }
        return FA_OK;
    });
}
