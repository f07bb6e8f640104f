// test_cond_host.cpp -- the null-handling members of the C++ host mirror (ScalarFunctions::{coalesce, greatest, least, nanvl},
// functions.hpp) on small columns of two chunks whose answers are exact.  Needs an H100; run by tests/test_cond_gpu.py (-m gpu).
#include <cmath>
#include <cstdio>
#include <cstring>
#include <limits>

#include "functions.hpp"

using namespace rdf;

static int g_failed = 0;
#define CHECK(cond) do { if (!(cond)) { std::printf("  FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); g_failed++; } } while (0)

static uint64_t bits_of(double x) { uint64_t b; std::memcpy(&b, &x, 8); return b; }

int main() {
    using O = std::optional<int32_t>;
    auto a0 = Int32Array::from(std::vector<O>{1, std::nullopt, std::nullopt});
    auto a1 = Int32Array::from(std::vector<O>{std::nullopt, 5});
    auto b0 = Int32Array::from(std::vector<O>{7, 8, std::nullopt});
    auto b1 = Int32Array::from(std::vector<O>{9, 2});
    const std::vector<const Int32Array*> a{&a0, &a1}, b{&b0, &b1};
    auto c = ScalarFunctions::coalesce<int32_t>({a, b});
    CHECK(c.is_ok() && c.unwrap().size() == 2);
    if (c.is_ok()) {
        const auto& r = c.unwrap();
        CHECK(r[0].value(0) == 1 && r[0].value(1) == 8 && r[0].is_null(2) && r[0].null_count() == 1);
        CHECK(r[1].value(0) == 9 && r[1].value(1) == 5 && r[1].null_count() == 0);
    }
    auto g = ScalarFunctions::greatest<int32_t>({a, b});
    auto l = ScalarFunctions::least<int32_t>({a, b});
    CHECK(g.is_ok() && l.is_ok());
    if (g.is_ok() && l.is_ok()) {
        CHECK(g.unwrap()[0].value(0) == 7 && g.unwrap()[0].value(1) == 8 && g.unwrap()[0].is_null(2) && g.unwrap()[1].value(1) == 5);
        CHECK(l.unwrap()[0].value(0) == 1 && l.unwrap()[1].value(0) == 9 && l.unwrap()[1].value(1) == 2);
    }
    // nanvl: a unless NaN, then b; NULL where a is NULL; the bits of the value taken
    const double nan = std::numeric_limits<double>::quiet_NaN();
    auto x = Float64Array::from(std::vector<std::optional<double>>{nan, -0.0, std::nullopt, nan});
    auto y = Float64Array::from(std::vector<std::optional<double>>{2.5, 1.0, 3.0, std::nullopt});
    auto n = ScalarFunctions::nanvl<double>({&x}, {&y});
    CHECK(n.is_ok());
    if (n.is_ok()) {
        const auto& r = n.unwrap()[0];
        CHECK(r.value(0) == 2.5 && bits_of(r.value(1)) == bits_of(-0.0) && r.is_null(2) && r.is_null(3) && r.null_count() == 2);
    }
    bool refused = false;   // nanvl of integers: T::Native: Float
    try { ScalarFunctions::nanvl<int32_t>(a, b); } catch (const std::logic_error&) { refused = true; }
    CHECK(refused);
    std::printf(g_failed ? "FAILED %d\n" : "COND OK\n", g_failed);
    return g_failed ? 1 : 0;
}
