// entry_guard.h — the message behind gb_last_error() and the one exception guard of the C entry points.
// Plain C++ without CUDA: the host-only units (emit.cpp, index_builder.cpp, gbz_reader.cpp) include it as the .cu units do.
#pragma once
#include "giraffe_b200.h"

#include <exception>
#include <new>
#include <string>

namespace gb {

// What the last failing call on this thread says went wrong (gb_last_error()).
inline thread_local std::string g_last_error;

// Sets g_last_error to a + b + c.  Never throws: when even that allocation fails the message is left empty.
inline void set_last_error(const char* a, const char* b, const char* c = "") noexcept {
    try { g_last_error.assign(a).append(b).append(c); } catch (...) { g_last_error.clear(); }
}

// Runs the body of the extern "C" entry point `entry` so that no exception leaves it (the policy is stated next to the status
// codes in giraffe_b200.h): std::bad_alloc becomes GB_ERR_CAPACITY, any other exception `other`.  `on_fail` runs first on
// either path; the readers clear their output handle there.
template <typename Body, typename OnFail>
int guarded(const char* entry, int other, Body&& body, OnFail&& on_fail) noexcept {
    try {
        return body();
    } catch (const std::bad_alloc&) {
        on_fail();
        set_last_error(entry, ": out of host memory");
        return GB_ERR_CAPACITY;
    } catch (const std::exception& e) {
        on_fail();
        set_last_error(e.what(), "");
        return other;
    } catch (...) {
        on_fail();
        set_last_error(entry, ": unknown exception");
        return other;
    }
}

template <typename Body>
int guarded(const char* entry, Body&& body) noexcept { return guarded(entry, GB_ERR_ARG, body, [] {}); }

} // namespace gb
