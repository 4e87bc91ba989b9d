// The host code's tuning knobs from the environment (a header of its own: the pass planner and its host-only test
// read them without the rest of the library)
#pragma once
#include <cstdlib>
#include <mutex>
#include <string>
#include <utility>
#include <vector>

// Tuning knobs from the environment.  FIDGET_B200_ENV_LIVE=1 re-reads them on every call (tests flip knobs
// between renders); otherwise each (name) is read once per process -- no getenv on the render path.
inline int env_int(const char* name, int dflt) {
    struct Slot { const char* name; int value; bool set; };
    static Slot cache[32];
    static std::mutex mu;
    static const bool live = [] { const char* v = getenv("FIDGET_B200_ENV_LIVE"); return v && *v && atoi(v) != 0; }();
    auto read = [&](int d) { const char* v = getenv(name); return v && *v ? atoi(v) : d; };
    if (live) return read(dflt);
    std::lock_guard<std::mutex> g(mu);
    for (auto& sl : cache) {
        if (sl.name == name) return sl.set ? sl.value : dflt;
        if (!sl.name) {
            const char* v = getenv(name);
            sl.name = name;
            sl.set = v && *v;
            sl.value = sl.set ? atoi(v) : 0;
            return sl.set ? sl.value : dflt;
        }
    }
    return read(dflt);
}
// String knobs, read like env_int: once per process, or on every call with FIDGET_B200_ENV_LIVE=1
inline std::string env_str(const char* name) {
    static std::mutex mu;
    static std::vector<std::pair<const char*, std::string>> cache;
    static const bool live = [] { const char* v = getenv("FIDGET_B200_ENV_LIVE"); return v && *v && atoi(v) != 0; }();
    auto read = [&] { const char* v = getenv(name); return std::string(v ? v : ""); };
    if (live) return read();
    std::lock_guard<std::mutex> g(mu);
    for (auto& kv : cache) if (kv.first == name) return kv.second;
    cache.emplace_back(name, read());
    return cache.back().second;
}
