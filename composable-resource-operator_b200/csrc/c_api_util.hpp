// c_api_util.hpp — small helpers shared by the extern "C" translation units (c_api.cu, harness.cu).
#pragma once

#include <cstdio>
#include <cstring>
#include <map>
#include <string>

#include "../../include/croprobe.h"

namespace cro {
namespace capi {


// Copies a text out through a caller-allocated buffer.  *len always receives the FULL length; when the buffer is too
// small the caller still gets a NUL-terminated prefix (never stale bytes from an earlier call) and CRO_ERR_BUFFER_SMALL.
inline int copy_out(const std::string& s, char* buf, size_t cap, size_t* len) {
    if (len) *len = s.size();
    if (!buf || cap == 0) return CRO_ERR_BUFFER_SMALL;
    if (cap < s.size() + 1) {
        memcpy(buf, s.data(), cap - 1);
        buf[cap - 1] = '\0';
        return CRO_ERR_BUFFER_SMALL;
    }
    memcpy(buf, s.data(), s.size());
    buf[s.size()] = '\0';
    return CRO_OK;
}

inline std::string S(const char* p) { return p ? std::string(p) : std::string(); }

inline std::string fixed_str(const char* p, size_t cap) { return std::string(p, strnlen(p, cap)); }

// bytes per ns == GB/s; one decimal, integer arithmetic only.
inline std::string gbs_x10(uint64_t bytes, uint64_t ns) {
    if (ns == 0) return "0.0";
    const unsigned __int128 v = (unsigned __int128)bytes * 10u / ns;
    const uint64_t q = (uint64_t)v;
    return std::to_string(q / 10) + "." + std::to_string(q % 10);
}

inline std::string hex16(uint64_t v) {
    char b[24];
    snprintf(b, sizeof b, "%016llx", (unsigned long long)v);
    return b;
}

// No C++ exception may cross the C ABI (the caller is cgo / ctypes: unwinding into it is undefined).  Every
// `int cro_*` entry point is a function-try-block ending in CRO_API_CATCH; on_exception() rethrows to classify:
// std::bad_alloc -> CRO_ERR_OOM, anything else -> CRO_ERR_INTERNAL, the what() text kept for the calling thread
// (cro_last_error(NULL, ...)).  Defined in c_api.cu.
int on_exception() noexcept;
#define CRO_API_CATCH catch (...) { return ::cro::capi::on_exception(); }

// The least sms_covered over the legs run: the "sms" annotation's numerator and what makes a health check incomplete;
// 0 when no leg ran.
template <class Leg>
uint32_t min_covered(uint32_t legs, const Leg* leg, int n_legs) {
    uint32_t covered = 0xFFFFFFFFu;
    for (int l = 0; l < n_legs; ++l)
        if (legs >> l & 1u) covered = covered < leg[l].sms_covered ? covered : leg[l].sms_covered;
    return covered == 0xFFFFFFFFu ? 0u : covered;
}

// cohdi.io/probe-* annotations of one result (defined in c_api.cu)
std::map<std::string, std::string> probe_annotations(const cro_probe_result& r);

}  // namespace capi
}  // namespace cro
