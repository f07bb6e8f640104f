// test_stats_host.cpp -- the statistical members of the C++ host mirror (AggregateFunctions::{variance, variance_pop, stddev,
// stddev_pop, skewness, kurtosis, count_distinct, sum_distinct}, functions.hpp) on small columns whose answers are exact.
// Needs an H100; run by tests/test_stats_gpu.py (-m gpu).
#include <cmath>
#include <cstdio>
#include <limits>

#include "functions.hpp"

using namespace rdf;

static const double EPS = std::numeric_limits<double>::epsilon();

static int g_failed = 0;
#define CHECK(cond) do { if (!(cond)) { std::printf("  FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); g_failed++; } } while (0)

int main() {
    // 1, 2, 3, 4 and a null: mean 2.5, m2 = 5, m3 = 0, m4 = 10.25 (the record is merged from per-thread pieces, so within a few ulp)
    auto a = Float64Array::from(std::vector<std::optional<double>>{1.0, std::nullopt, 2.0});
    auto b = Float64Array::from(std::vector<double>{3.0, 4.0});
    const std::vector<const Float64Array*> ab{&a, &b};
    auto near = [](std::optional<double> got, double want) { return got && std::fabs(*got - want) <= 64 * EPS * std::fabs(want); };
    CHECK(near(AggregateFunctions::variance<double>(ab), 5.0 / 3.0));
    CHECK(near(AggregateFunctions::variance_pop<double>(ab), 1.25));
    CHECK(near(AggregateFunctions::stddev<double>(ab), std::sqrt(5.0 / 3.0)));
    CHECK(near(AggregateFunctions::stddev_pop<double>(ab), std::sqrt(1.25)));
    const auto skew = AggregateFunctions::skewness<double>(ab);
    CHECK(skew && std::fabs(*skew) <= 1e-14);
    CHECK(near(AggregateFunctions::kurtosis<double>(ab), (4.0 * 10.25) / 25.0 - 3.0));

    // None rules: one value has no sample variance; a constant column has no skewness
    auto one = Int64Array::from(std::vector<int64_t>{7});
    CHECK(!AggregateFunctions::variance<int64_t>({&one}).has_value());
    CHECK(AggregateFunctions::variance_pop<int64_t>({&one}) == 0.0);
    auto c = Float64Array::from(std::vector<double>{0.1, 0.1, 0.1});
    CHECK(AggregateFunctions::stddev<double>({&c}) == 0.0);
    CHECK(!AggregateFunctions::skewness<double>({&c}).has_value());
    CHECK(!AggregateFunctions::kurtosis<double>({&c}).has_value());

    // distinct: -0.0 == 0.0 and every NaN is one value; nulls are not counted
    const double nan = std::numeric_limits<double>::quiet_NaN();
    auto d = Float64Array::from(std::vector<std::optional<double>>{1.5, -0.0, 0.0, std::nullopt, 1.5, 2.0});
    CHECK(AggregateFunctions::count_distinct<double>({&d}) == 3);
    CHECK(AggregateFunctions::sum_distinct<double>({&d}) == 3.5);
    auto e = Float64Array::from(std::vector<double>{nan, -nan, 1.0});
    CHECK(AggregateFunctions::count_distinct<double>({&e}) == 2);
    CHECK(std::isnan(AggregateFunctions::sum_distinct<double>({&e})));
    auto i = Int32Array::from(std::vector<int32_t>{2147483647, 1, 2147483647, 1});
    CHECK(AggregateFunctions::sum_distinct<int32_t>({&i}) == (int32_t)0x80000000);   // wraps
    auto none = Int32Array::from(std::vector<std::optional<int32_t>>{std::nullopt});
    CHECK(AggregateFunctions::sum_distinct<int32_t>({&none}) == 0 && AggregateFunctions::count_distinct<int32_t>({&none}) == 0);

    std::printf(g_failed ? "FAILED %d\n" : "STATS OK\n", g_failed);
    return g_failed ? 1 : 0;
}
