// civil.cuh -- the proleptic Gregorian calendar of the temporal functions (k_temporal.cu) and the JSON writer's dates
// (json_format.cuh): chrono's day range and Hinnant's civil_from_days ("chrono-Compatible Low-Level Date Algorithms", PAPERS.md).
// Plain integer arithmetic, so a host compiler (with __device__ defined empty) gives the same fields.
#pragma once

#include <stdint.h>

namespace bdf {

#if defined(__CUDACC__)
#define CIVILF __host__ __device__ __forceinline__
#else
#define CIVILF inline
#endif

constexpr int32_t kMinDay = -96465658;   // -262144-01-01, chrono's NaiveDate::MIN
constexpr int32_t kMaxDay = 95026601;    //  262143-12-31, chrono's NaiveDate::MAX

// Hinnant's civil_from_days on 32-bit integers (valid for every day of chrono's range).
CIVILF void civil_from_days(int32_t z, int32_t& y, uint32_t& m, uint32_t& d) {
    z += 719468;
    const int32_t era = (z >= 0 ? z : z - 146096) / 146097;
    const uint32_t doe = (uint32_t)(z - era * 146097);
    const uint32_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
    const uint32_t doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
    const uint32_t mp = (5 * doy + 2) / 153;
    d = doy - (153 * mp + 2) / 5 + 1;
    m = mp < 10 ? mp + 3 : mp - 9;
    y = (int32_t)yoe + era * 400 + (m <= 2 ? 1 : 0);
}

}  // namespace bdf
