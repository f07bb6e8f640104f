// test_dist_host.cpp -- the distribution members of the C++ host mirror (AggregateFunctions::{percentile, median, mode},
// functions.hpp) on small columns whose answers are exact.  Needs an H100; run by tests/test_distribution_gpu.py (-m gpu).
#include <cmath>
#include <cstdio>
#include <limits>

#include "functions.hpp"

using namespace rdf;

static int g_failed = 0;
#define CHECK(cond) do { if (!(cond)) { std::printf("  FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); g_failed++; } } while (0)

int main() {
    // 0..9 over two arrays with a null: the median interpolates at (n - 1) * 0.5
    auto a = Float64Array::from(std::vector<std::optional<double>>{3.0, std::nullopt, 0.0, 9.0, 1.0});
    auto b = Float64Array::from(std::vector<double>{2.0, 8.0, 4.0, 7.0, 5.0, 6.0});
    const std::vector<const Float64Array*> ab{&a, &b};
    CHECK(AggregateFunctions::median<double>(ab) == 4.5);
    CHECK(AggregateFunctions::percentile<double>(ab, 0.0) == 0.0 && AggregateFunctions::percentile<double>(ab, 1.0) == 9.0);
    CHECK(AggregateFunctions::percentile<double>(ab, 0.25) == 2.25);
    // mode: the most frequent value, ties to the smallest; -0.0 == 0.0; None without a valid value
    auto i = Int32Array::from(std::vector<int32_t>{9, 4, 9, 4, 1});
    CHECK(AggregateFunctions::mode<int32_t>({&i}) == 4);
    auto z = Float64Array::from(std::vector<double>{-0.0, 0.0, 2.0});
    const auto m = AggregateFunctions::mode<double>({&z});
    CHECK(m && *m == 0.0 && std::signbit(*m));   // the class's first row
    auto none = Int64Array::from(std::vector<std::optional<int64_t>>{std::nullopt, std::nullopt});
    CHECK(!AggregateFunctions::mode<int64_t>({&none}).has_value() && !AggregateFunctions::median<int64_t>({&none}).has_value());
    // a NaN majority: the median is the positive quiet NaN
    const double nan = std::numeric_limits<double>::quiet_NaN();
    auto n = Float64Array::from(std::vector<double>{nan, -nan, nan, 1.0});
    const auto med = AggregateFunctions::median<double>({&n});
    uint64_t bits = 0;
    if (med) std::memcpy(&bits, &*med, 8);
    CHECK(med && bits == 0x7ff8000000000000ull);
    bool refused = false;
    try { AggregateFunctions::percentile<double>(ab, 1.5); } catch (const std::runtime_error&) { refused = true; }
    CHECK(refused);
    std::printf(g_failed ? "FAILED %d\n" : "DIST OK\n", g_failed);
    return g_failed ? 1 : 0;
}
