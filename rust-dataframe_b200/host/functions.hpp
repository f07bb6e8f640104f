// functions.hpp -- C++ host mirror of the reference's operator interface for the hot path, one C-ABI call
// (libb200df.so, include/b200df.h) per function.  Same names, argument meaning and error behaviour as
//   ScalarFunctions     reference src/functions/scalar.rs:14-497
//   AggregateFunctions  reference src/functions/aggregate.rs:9-103
//   cast                the arrow::compute::cast call of Function::Cast, src/evaluation.rs:296-315
// so that tests written against the reference read the same here.  Nothing in this file computes: values
// are produced by the CUDA kernels behind the ABI.  The Rust binding a maintainer would add has exactly
// this shape (INTEGRATION.md).
#pragma once

#include <algorithm>
#include <cstring>
#include <optional>
#include <string>
#include <utility>
#include <variant>
#include <vector>

#include "b200df.h"
#include "primitive_array.hpp"

namespace rdf {

// arrow::error::ArrowError (the variants the hot path can produce)
struct ArrowError {
    enum Kind { ComputeError, DivideByZero } kind;
    std::string message;
    std::string to_string() const { return kind == DivideByZero ? "Divide by zero error" : "Compute error: " + message; }
};

struct ReferencePanic : std::runtime_error {  // where the Rust reference panics (unwrap on None, bad downcast)
    using std::runtime_error::runtime_error;
};

// Result<T, ArrowError>
template <typename T>
class Result {
   public:
    Result(T v) : v_(std::move(v)) {}
    Result(ArrowError e) : v_(std::move(e)) {}
    bool is_ok() const { return std::holds_alternative<T>(v_); }
    bool is_err() const { return !is_ok(); }
    T& unwrap() {
        if (is_err()) throw ReferencePanic("called `Result::unwrap()` on an `Err` value: " + std::get<ArrowError>(v_).to_string());
        return std::get<T>(v_);
    }
    const ArrowError& unwrap_err() const { return std::get<ArrowError>(v_); }

   private:
    std::variant<T, ArrowError> v_;
};

// Process-wide context, created on first use (what the Rust shim keeps in a Once, integration/rust/src/ffi.rs `ctx()`): ONE
// context over every GPU of the box (bdf_init_multi: the library shards each call by row range, the job rayon's par_iter does in
// src/functions/scalar.rs:28-31,99-102) -- unless a process-per-GPU launcher started this process (WORLD_SIZE > 1: GPU LOCAL_RANK,
// the job is joined with bdf_comm_attach) or BDF_ONE_GPU is set.
inline bdf_ctx* context() {
    static bdf_ctx* ctx = [] {
        bdf_ctx* c = nullptr;
        const char* ws = std::getenv("WORLD_SIZE");
        const char* lr = std::getenv("LOCAL_RANK");
        const bool one = (ws && std::atoi(ws) > 1) || std::getenv("BDF_ONE_GPU");
        const int st = one ? bdf_init(lr ? std::atoi(lr) : 0, &c) : bdf_init_multi(0, nullptr, &c);
        if (st != BDF_OK) throw std::runtime_error(std::string("libb200df initialisation failed: ") + bdf_last_error());
        return c;
    }();
    return ctx;
}

namespace detail {

inline ArrowError to_error(int st) {
    if (st == BDF_DIVIDE_BY_ZERO) return {ArrowError::DivideByZero, ""};
    if (st == BDF_LENGTH_MISMATCH) return {ArrowError::ComputeError, "Cannot perform math operation on arrays of different length"};
    return {ArrowError::ComputeError, bdf_last_error()};
}

template <typename T>
std::vector<bdf_view> views(const std::vector<const PrimitiveArray<T>*>& arrays) {
    std::vector<bdf_view> v;
    v.reserve(arrays.size());
    for (auto* a : arrays) v.push_back(a->view());
    return v;
}

template <typename T>
struct Outputs {
    std::vector<std::shared_ptr<Buffer>> values, validity;
    std::vector<bdf_out> outs;
    explicit Outputs(const std::vector<int64_t>& lens) {
        for (int64_t n : lens) {
            values.push_back(std::make_shared<Buffer>(size_t(n) * sizeof(T)));       // MutableBuffer::new(n * size_of::<T>())
            validity.push_back(std::make_shared<Buffer>(size_t(n + 7) / 8));
            bdf_out o{values.back()->data(), validity.back()->data(), n, 0, 0};
            outs.push_back(o);
        }
    }
    std::vector<PrimitiveArray<T>> finish() {
        std::vector<PrimitiveArray<T>> res;
        for (size_t i = 0; i < outs.size(); i++)
            res.push_back(PrimitiveArray<T>::from_buffers(values[i], outs[i].has_validity ? validity[i] : nullptr, outs[i].len,
                                                           outs[i].has_validity ? outs[i].null_count : 0));
        return res;
    }
};

template <typename T>
Result<std::vector<PrimitiveArray<T>>> binary(int op, const std::vector<const PrimitiveArray<T>*>& left,
                                              const std::vector<const PrimitiveArray<T>*>& right) {
    const size_t n = std::min(left.size(), right.size());  // zip()
    std::vector<int64_t> lens;
    for (size_t i = 0; i < n; i++) lens.push_back(left[i]->len());
    Outputs<T> out(lens);
    auto lv = views(left), rv = views(right);
    const int st = bdf_binary(context(), op, ArrowType<T>::id, (int64_t)lv.size(), lv.data(), (int64_t)rv.size(), rv.data(), out.outs.data());
    if (st == BDF_UNSUPPORTED) throw std::logic_error(std::string("trait bound not satisfied: ") + bdf_last_error());
    if (st != BDF_OK) return to_error(st);
    return out.finish();
}

template <typename T>
Result<std::vector<PrimitiveArray<T>>> unary(int op, const std::vector<const PrimitiveArray<T>*>& array) {
    std::vector<int64_t> lens;
    for (auto* a : array) lens.push_back(a->len());
    Outputs<T> out(lens);
    auto v = views(array);
    const int st = bdf_unary(context(), op, ArrowType<T>::id, (int64_t)v.size(), v.data(), out.outs.data());
    if (st == BDF_UNSUPPORTED) throw std::logic_error(std::string("trait bound not satisfied: ") + bdf_last_error());
    if (st != BDF_OK) return to_error(st);
    return out.finish();
}

// Dates and timestamps: T is the column's physical type (int32_t / int64_t), R the result's (bdf_temporal_result says which).
template <typename T, typename R>
Result<std::vector<PrimitiveArray<R>>> temporal(int fn, const bdf_temporal_type& type, int64_t arg, const std::vector<const PrimitiveArray<T>*>& array) {
    int32_t dt = -1;
    int st = bdf_temporal_result(fn, &type, arg, &dt, nullptr);
    if (st == BDF_UNSUPPORTED) throw std::logic_error(std::string("temporal function not available: ") + bdf_last_error());
    if (st != BDF_OK) return to_error(st);
    if (dt != ArrowType<R>::id) throw std::logic_error("the result type R does not match bdf_temporal_result");
    std::vector<int64_t> lens;
    for (auto* a : array) lens.push_back(a->len());
    Outputs<R> out(lens);
    auto v = views(array);
    st = bdf_temporal(context(), fn, &type, arg, (int64_t)v.size(), v.data(), out.outs.data());
    if (st == BDF_UNSUPPORTED) throw std::logic_error(std::string("temporal function not available: ") + bdf_last_error());
    if (st != BDF_OK) return to_error(st);
    return out.finish();
}

// Null handling and conditional selection over host chunks: every column is uploaded, the device entry runs on them, the result
// comes back.  zip() semantics as the device entry has them: the smallest chunk count of the columns.
template <typename T>
Result<std::vector<PrimitiveArray<T>>> rowwise(int fn, const std::vector<std::vector<const PrimitiveArray<T>*>>& columns) {
    std::vector<bdf_col*> cols;
    std::vector<bdf_arg> args;
    auto release = [&] { for (auto* c : cols) bdf_col_free(context(), c); };
    size_t n = columns.empty() ? 0 : columns[0].size();
    for (auto& c : columns) n = std::min(n, c.size());
    int st = BDF_OK;
    for (auto& c : columns) {
        auto v = views(c);
        bdf_col* col = nullptr;
        st = bdf_upload(context(), ArrowType<T>::id, (int64_t)v.size(), v.data(), 0, &col);
        if (st != BDF_OK) break;
        cols.push_back(col);
        args.push_back(bdf_arg{col, 0, 1});
    }
    bdf_col* res = nullptr;
    if (st == BDF_OK) st = bdf_rowwise_dev(context(), fn, (int32_t)args.size(), args.data(), &res);
    if (st == BDF_UNSUPPORTED) { release(); throw std::logic_error(std::string("trait bound not satisfied: ") + bdf_last_error()); }
    if (st != BDF_OK) { release(); return to_error(st); }
    std::vector<int64_t> lens;
    for (size_t i = 0; i < n; i++) lens.push_back(columns[0][i]->len());
    Outputs<T> out(lens);
    st = bdf_download(context(), res, out.outs.data());
    bdf_col_free(context(), res);
    release();
    if (st != BDF_OK) return to_error(st);
    return out.finish();
}

}  // namespace detail

struct ScalarFunctions {
    template <typename T> using Arrays = std::vector<const PrimitiveArray<T>*>;  // Vec<&PrimitiveArray<T>>
    template <typename T> using Out = Result<std::vector<PrimitiveArray<T>>>;    // Result<Vec<PrimitiveArray<T>>, ArrowError>

    template <typename T> static Out<T> add(const Arrays<T>& l, const Arrays<T>& r) { return detail::binary<T>(BDF_ADD, l, r); }
    template <typename T> static Out<T> subtract(const Arrays<T>& l, const Arrays<T>& r) { return detail::binary<T>(BDF_SUB, l, r); }
    template <typename T> static Out<T> multiply(const Arrays<T>& l, const Arrays<T>& r) { return detail::binary<T>(BDF_MUL, l, r); }
    template <typename T> static Out<T> par_multiply(const Arrays<T>& l, const Arrays<T>& r) { return detail::binary<T>(BDF_MUL, l, r); }
    template <typename T> static Out<T> divide(const Arrays<T>& l, const Arrays<T>& r) { return detail::binary<T>(BDF_DIV, l, r); }

#define RDF_UNARY(name, OP) \
    template <typename T> static Out<T> name(const Arrays<T>& a) { return detail::unary<T>(OP, a); }
    RDF_UNARY(abs, BDF_ABS) RDF_UNARY(sin, BDF_SIN) RDF_UNARY(cos, BDF_COS) RDF_UNARY(tan, BDF_TAN) RDF_UNARY(acos, BDF_ACOS)
    RDF_UNARY(asin, BDF_ASIN) RDF_UNARY(atan, BDF_ATAN) RDF_UNARY(cbrt, BDF_CBRT) RDF_UNARY(ceil, BDF_CEIL)
    RDF_UNARY(cosh, BDF_COSH) RDF_UNARY(degrees, BDF_DEGREES) RDF_UNARY(exp, BDF_EXP) RDF_UNARY(expm1, BDF_EXPM1)
    RDF_UNARY(floor, BDF_FLOOR) RDF_UNARY(log10, BDF_LOG10) RDF_UNARY(log2, BDF_LOG2) RDF_UNARY(radians, BDF_RADIANS)
    RDF_UNARY(round, BDF_ROUND) RDF_UNARY(sinh, BDF_SINH) RDF_UNARY(sqrt, BDF_SQRT) RDF_UNARY(tanh, BDF_TANH)
#undef RDF_UNARY

    // Dates and timestamps (include/b200df.h "dates and timestamps"): `type` is the Arrow temporal type of the column of physical T.
    // ScalarFunctions::hour<T>(Vec<&PrimitiveArray<T>>) -> Vec<Int32Array> (scalar.rs:267-273) and the stubs of the same file.
#define RDF_TEMPORAL(name, FN, R) \
    template <typename T> static Out<R> name(const bdf_temporal_type& t, const Arrays<T>& a) { return detail::temporal<T, R>(FN, t, 0, a); }
#define RDF_TEMPORAL_ARG(name, FN, R) \
    template <typename T> static Out<R> name(const bdf_temporal_type& t, int64_t arg, const Arrays<T>& a) { return detail::temporal<T, R>(FN, t, arg, a); }
    RDF_TEMPORAL(year, BDF_TEMPORAL_YEAR, int32_t) RDF_TEMPORAL(quarter, BDF_TEMPORAL_QUARTER, int32_t) RDF_TEMPORAL(month, BDF_TEMPORAL_MONTH, int32_t)
    RDF_TEMPORAL(day_of_month, BDF_TEMPORAL_DAY_OF_MONTH, int32_t) RDF_TEMPORAL(day_of_year, BDF_TEMPORAL_DAY_OF_YEAR, int32_t)
    RDF_TEMPORAL(day_of_week, BDF_TEMPORAL_DAY_OF_WEEK, int32_t) RDF_TEMPORAL(hour, BDF_TEMPORAL_HOUR, int32_t)
    RDF_TEMPORAL(minute, BDF_TEMPORAL_MINUTE, int32_t) RDF_TEMPORAL(second, BDF_TEMPORAL_SECOND, int32_t)
    RDF_TEMPORAL(to_date, BDF_TEMPORAL_TO_DATE, int32_t) RDF_TEMPORAL(last_day, BDF_TEMPORAL_LAST_DAY, int32_t)
    RDF_TEMPORAL(unix_timestamp, BDF_TEMPORAL_UNIX_TIMESTAMP, int64_t)
    RDF_TEMPORAL_ARG(date_add, BDF_TEMPORAL_DATE_ADD, int32_t) RDF_TEMPORAL_ARG(date_sub, BDF_TEMPORAL_DATE_SUB, int32_t)
    RDF_TEMPORAL_ARG(add_months, BDF_TEMPORAL_ADD_MONTHS, int32_t) RDF_TEMPORAL_ARG(next_day, BDF_TEMPORAL_NEXT_DAY, int32_t)
    RDF_TEMPORAL_ARG(to_timestamp, BDF_TEMPORAL_TO_TIMESTAMP, int64_t)
#undef RDF_TEMPORAL
#undef RDF_TEMPORAL_ARG
    // coalesce / greatest / least / nanv1: scalar.rs's empty stubs with Spark's definitions (include/b200df.h "null handling and
    // conditional selection"); every argument is a column given as its chunks.
    template <typename T> static Out<T> coalesce(const std::vector<Arrays<T>>& a) { return detail::rowwise<T>(BDF_ROW_COALESCE, a); }
    template <typename T> static Out<T> greatest(const std::vector<Arrays<T>>& a) { return detail::rowwise<T>(BDF_ROW_GREATEST, a); }
    template <typename T> static Out<T> least(const std::vector<Arrays<T>>& a) { return detail::rowwise<T>(BDF_ROW_LEAST, a); }
    template <typename T> static Out<T> nanvl(const Arrays<T>& a, const Arrays<T>& b) { return detail::rowwise<T>(BDF_ROW_NANVL, {a, b}); }
    // date_trunc keeps the input's type: the result has the column's physical type T
    template <typename T> static Out<T> date_trunc(const bdf_temporal_type& t, int64_t unit, const Arrays<T>& a) {
        return detail::temporal<T, T>(BDF_TEMPORAL_DATE_TRUNC, t, unit, a);
    }
};

// arrow::compute::cast over every chunk of a column (Function::Cast, src/evaluation.rs:296-315)
template <typename From, typename To>
Result<std::vector<PrimitiveArray<To>>> cast(const std::vector<const PrimitiveArray<From>*>& arrays) {
    std::vector<int64_t> lens;
    for (auto* a : arrays) lens.push_back(a->len());
    detail::Outputs<To> out(lens);
    auto v = detail::views(arrays);
    const int st = bdf_cast(context(), ArrowType<From>::id, ArrowType<To>::id, (int64_t)v.size(), v.data(), out.outs.data());
    if (st != BDF_OK) return detail::to_error(st);
    return out.finish();
}

struct AggregateFunctions {
    template <typename T> using Arrays = std::vector<const PrimitiveArray<T>*>;

    template <typename T> static std::optional<T> sum(const Arrays<T>& a) { return agg<T, T>(BDF_SUM, a); }
    template <typename T> static std::optional<T> max(const Arrays<T>& a) { return agg<T, T>(BDF_MAX, a); }
    // The reference's min is a copy of max (aggregate.rs:22-31); this is the intended min.
    template <typename T> static std::optional<T> min(const Arrays<T>& a) { return agg<T, T>(BDF_MIN, a); }
    template <typename T> static std::optional<int64_t> count(const Arrays<T>& a) { return agg<T, int64_t>(BDF_COUNT, a); }
    template <typename T> static std::optional<double> avg(const Arrays<T>& a) {
        auto v = detail::views(a);
        double out = 0; int32_t some = 0;
        check(bdf_avg(context(), ArrowType<T>::id, (int64_t)v.size(), v.data(), &out, &some));
        return some ? std::optional<double>(out) : std::nullopt;
    }
    // The stubs of aggregate.rs:81,94-102 (include/b200df.h "statistical aggregates"): sample variance / stddev as Spark's, the
    // population forms, skewness, excess kurtosis; any numeric T, read as f64.
    template <typename T> static std::optional<double> variance(const Arrays<T>& a) { return stat<T>(BDF_STAT_VARIANCE, a); }
    template <typename T> static std::optional<double> variance_pop(const Arrays<T>& a) { return stat<T>(BDF_STAT_VAR_POP, a); }
    template <typename T> static std::optional<double> stddev(const Arrays<T>& a) { return stat<T>(BDF_STAT_STDDEV, a); }
    template <typename T> static std::optional<double> stddev_pop(const Arrays<T>& a) { return stat<T>(BDF_STAT_STDDEV_POP, a); }
    template <typename T> static std::optional<double> skewness(const Arrays<T>& a) { return stat<T>(BDF_STAT_SKEWNESS, a); }
    template <typename T> static std::optional<double> kurtosis(const Arrays<T>& a) { return stat<T>(BDF_STAT_KURTOSIS, a); }
    template <typename T> static int64_t count_distinct(const Arrays<T>& a) { return distinct<T>(a).count; }
    template <typename T> static T sum_distinct(const Arrays<T>& a) {   // 0 without a valid value, like sum
        const bdf_distinct_rec r = distinct<T>(a);
        T out{};
        std::memcpy(&out, &r.sum, sizeof(T));
        return out;
    }
    // The distributions (include/b200df.h "distributions"): Spark's exact percentile (p in [0, 1]), median and mode.
    template <typename T> static std::optional<double> percentile(const Arrays<T>& a, double p) {
        auto v = detail::views(a);
        double out = 0; int32_t some = 0;
        check(bdf_percentile(context(), ArrowType<T>::id, (int64_t)v.size(), v.data(), 1, &p, &out, &some));
        return some ? std::optional<double>(out) : std::nullopt;
    }
    template <typename T> static std::optional<double> median(const Arrays<T>& a) { return percentile<T>(a, 0.5); }
    template <typename T> static std::optional<T> mode(const Arrays<T>& a) {   // ties: the smallest value
        auto v = detail::views(a);
        uint64_t bits = 0; int64_t freq = 0; int32_t some = 0;
        check(bdf_mode(context(), ArrowType<T>::id, (int64_t)v.size(), v.data(), &bits, &freq, &some));
        if (!some) return std::nullopt;
        T out{};
        std::memcpy(&out, &bits, sizeof(T));
        return out;
    }

   private:
    template <typename T> static std::optional<double> stat(int which, const Arrays<T>& a) {
        auto v = detail::views(a);
        bdf_moment_rec m{};
        check(bdf_moments(context(), ArrowType<T>::id, (int64_t)v.size(), v.data(), &m));
        double out = 0; int32_t some = 0;
        check(bdf_moments_stat(&m, which, &out, &some));
        return some ? std::optional<double>(out) : std::nullopt;
    }
    template <typename T> static bdf_distinct_rec distinct(const Arrays<T>& a) {
        auto v = detail::views(a);
        bdf_distinct_rec r{};
        check(bdf_distinct(context(), ArrowType<T>::id, (int64_t)v.size(), v.data(), &r));
        return r;
    }
    static void check(int st) {
        if (st == BDF_WOULD_PANIC) throw ReferencePanic(bdf_last_error());
        if (st == BDF_UNSUPPORTED) throw std::logic_error(std::string("trait bound not satisfied: ") + bdf_last_error());
        if (st != BDF_OK) throw std::runtime_error(bdf_last_error());
    }
    template <typename T, typename R> static std::optional<R> agg(int op, const Arrays<T>& a) {
        auto v = detail::views(a);
        R out{}; int32_t some = 0;
        check(bdf_aggregate(context(), op, ArrowType<T>::id, (int64_t)v.size(), v.data(), &out, &some));
        return some ? std::optional<R>(out) : std::nullopt;
    }
};

}  // namespace rdf
