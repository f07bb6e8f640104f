//! Replacement bodies for src/functions/aggregate.rs (signatures unchanged).  UNCOMPILED here -- see ../README.md.
use std::os::raw::{c_int, c_void};

use arrow::array::PrimitiveArray;
use arrow::datatypes::ArrowNumericType;

use crate::ffi::*;

/// op: 0 sum, 1 min, 2 max, 3 count (bdf_aggop).  R = T::Native for sum/min/max, i64 for count.
pub fn gpu_agg<T: ArrowNumericType, R: Default>(op: c_int, arrays: &[&PrimitiveArray<T>]) -> Option<R> {
    let v: Vec<BdfView> = arrays.iter().map(|a| view(*a)).collect();
    let (mut out, mut some) = (R::default(), 0i32);
    let st = unsafe {
        bdf_aggregate(ctx(), op, dtype_id(&T::get_data_type()), v.len() as i64, v.as_ptr(), &mut out as *mut R as *mut c_void, &mut some)
    };
    match st {
        BDF_OK => if some != 0 { Some(out) } else { None },
        // the reference calls compute::max(array).unwrap() per chunk (aggregate.rs:19,29): None panics there too
        BDF_WOULD_PANIC => panic!("called `Option::unwrap()` on a `None` value"),
        st => panic!("{}", to_arrow_error(st)),
    }
}

pub fn gpu_avg<T: ArrowNumericType>(arrays: &[&PrimitiveArray<T>]) -> Option<f64> {
    let v: Vec<BdfView> = arrays.iter().map(|a| view(*a)).collect();
    let (mut out, mut some) = (0f64, 0i32);
    let st = unsafe { bdf_avg(ctx(), dtype_id(&T::get_data_type()), v.len() as i64, v.as_ptr(), &mut out, &mut some) };
    assert_eq!(st, BDF_OK, "{}", last_error());
    if some != 0 { Some(out) } else { None }
}

/// The statistic `stat` (bdf_stat) of the moment record of every chunk's valid values: None per include/b200df.h (count 0; count 1
/// for the sample forms; m2 == 0 for skewness / kurtosis).  Any numeric T (Int64 / UInt64 included), read `as f64`.
pub fn gpu_stat<T: ArrowNumericType>(stat: c_int, arrays: &[&PrimitiveArray<T>]) -> Option<f64> {
    let v: Vec<BdfView> = arrays.iter().map(|a| view(*a)).collect();
    let mut m = BdfMomentRec::default();
    let st = unsafe { bdf_moments(ctx(), dtype_id(&T::get_data_type()), v.len() as i64, v.as_ptr(), &mut m) };
    assert_eq!(st, BDF_OK, "{}", last_error());
    let (mut out, mut some) = (0f64, 0i32);
    let st = unsafe { bdf_moments_stat(&m, stat, &mut out, &mut some) };
    assert_eq!(st, BDF_OK, "{}", last_error());
    if some != 0 { Some(out) } else { None }
}

/// (count, sum) of the distinct valid values (all NaNs one value, -0.0 == 0.0); the sum is T::Native, 0 without a valid value.
pub fn gpu_distinct<T: ArrowNumericType>(arrays: &[&PrimitiveArray<T>]) -> (i64, T::Native) {
    let v: Vec<BdfView> = arrays.iter().map(|a| view(*a)).collect();
    let mut r = BdfDistinctRec::default();
    let st = unsafe { bdf_distinct(ctx(), dtype_id(&T::get_data_type()), v.len() as i64, v.as_ptr(), &mut r) };
    assert_eq!(st, BDF_OK, "{}", last_error());
    let sum = unsafe { std::ptr::read_unaligned(&r.sum as *const u64 as *const T::Native) };   // the low bytes, little endian
    (r.count, sum)
}

/// Spark's exact percentile of the valid values at p in [0, 1] (include/b200df.h "distributions"); None without a valid value.
pub fn gpu_percentile<T: ArrowNumericType>(arrays: &[&PrimitiveArray<T>], p: f64) -> Option<f64> {
    let v: Vec<BdfView> = arrays.iter().map(|a| view(*a)).collect();
    let (mut out, mut some) = (0f64, 0i32);
    let st = unsafe { bdf_percentile(ctx(), dtype_id(&T::get_data_type()), v.len() as i64, v.as_ptr(), 1, &p, &mut out, &mut some) };
    assert_eq!(st, BDF_OK, "{}", last_error());
    if some != 0 { Some(out) } else { None }
}

/// The most frequent valid value (ties: the smallest in the sort's order) and its row count; None without a valid value.
pub fn gpu_mode<T: ArrowNumericType>(arrays: &[&PrimitiveArray<T>]) -> Option<(T::Native, i64)> {
    let v: Vec<BdfView> = arrays.iter().map(|a| view(*a)).collect();
    let (mut bits, mut freq, mut some) = (0u64, 0i64, 0i32);
    let st = unsafe { bdf_mode(ctx(), dtype_id(&T::get_data_type()), v.len() as i64, v.as_ptr(), &mut bits, &mut freq, &mut some) };
    assert_eq!(st, BDF_OK, "{}", last_error());
    if some == 0 { return None; }
    Some((unsafe { std::ptr::read_unaligned(&bits as *const u64 as *const T::Native) }, freq))
}

// In src/functions/aggregate.rs:
//   pub fn sum<T>(arrays)   -> gpu_agg::<T, T::Native>(0, &arrays)
//   pub fn min<T>(arrays)   -> gpu_agg::<T, T::Native>(1, &arrays)   // the intended minimum; the current body is a copy of max (aggregate.rs:22-31)
//   pub fn max<T>(arrays)   -> gpu_agg::<T, T::Native>(2, &arrays)
//   pub fn count<T>(arrays) -> gpu_agg::<T, i64>(3, &arrays)         // metadata only when the null counts are known
//   pub fn avg<T>(arrays)   -> gpu_avg(&arrays)
//   pub fn variance<T: ArrowNumericType>(arrays: Vec<&PrimitiveArray<T>>) -> Option<f64>     -> gpu_stat(BDF_STAT_VARIANCE, &arrays)   // sample, as Spark
//   pub fn variance_pop<T: ArrowNumericType>(arrays: Vec<&PrimitiveArray<T>>) -> Option<f64> -> gpu_stat(BDF_STAT_VAR_POP, &arrays)
//   pub fn stddev<T: ArrowNumericType>(arrays: Vec<&PrimitiveArray<T>>) -> Option<f64>       -> gpu_stat(BDF_STAT_STDDEV, &arrays)     // sample
//   pub fn stddev_pop<T: ArrowNumericType>(arrays: Vec<&PrimitiveArray<T>>) -> Option<f64>   -> gpu_stat(BDF_STAT_STDDEV_POP, &arrays)
//   pub fn skewness<T: ArrowNumericType>(arrays: Vec<&PrimitiveArray<T>>) -> Option<f64>     -> gpu_stat(BDF_STAT_SKEWNESS, &arrays)
//   pub fn kurtosis<T: ArrowNumericType>(arrays: Vec<&PrimitiveArray<T>>) -> Option<f64>     -> gpu_stat(BDF_STAT_KURTOSIS, &arrays)   // excess
//   pub fn count_distinct<T: ArrowNumericType>(arrays: Vec<&PrimitiveArray<T>>) -> i64       -> gpu_distinct(&arrays).0
//   pub fn sum_distinct<T: ArrowNumericType>(arrays: Vec<&PrimitiveArray<T>>) -> T::Native   -> gpu_distinct(&arrays).1    // 0, not None, like sum
//   pub fn percentile<T: ArrowNumericType>(arrays: Vec<&PrimitiveArray<T>>, p: f64) -> Option<f64> -> gpu_percentile(&arrays, p)
//   pub fn median<T: ArrowNumericType>(arrays: Vec<&PrimitiveArray<T>>) -> Option<f64>       -> gpu_percentile(&arrays, 0.5)
//   pub fn mode<T: ArrowNumericType>(arrays: Vec<&PrimitiveArray<T>>) -> Option<T::Native>   -> gpu_mode(&arrays).map(|m| m.0)
