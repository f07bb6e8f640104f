//! Replacement bodies for src/functions/scalar.rs (signatures unchanged).  UNCOMPILED here -- see ../README.md.
use std::os::raw::{c_int, c_void};
use std::sync::Arc;

use arrow::array::{Array, ArrayData, PrimitiveArray};
use arrow::buffer::MutableBuffer;
use arrow::datatypes::{ArrowNumericType, ArrowPrimitiveType, DataType, DateUnit, TimeUnit};
use arrow::error::ArrowError;

use crate::ffi::*;

/// op: 0 add, 1 subtract, 2 multiply, 3 divide, 4 atan2, 5 hypot, 6 log (bdf_binop)
pub fn gpu_binary<T: ArrowNumericType>(op: c_int, left: Vec<&PrimitiveArray<T>>, right: Vec<&PrimitiveArray<T>>)
    -> Result<Vec<PrimitiveArray<T>>, ArrowError>
{
    let n = left.len().min(right.len()); // zip()
    let lv: Vec<BdfView> = left.iter().map(|a| view(*a)).collect();
    let rv: Vec<BdfView> = right.iter().map(|a| view(*a)).collect();
    let (vals, bits, mut outs) = alloc_outputs::<T>(&left[..n].iter().map(|a| a.len()).collect::<Vec<_>>());
    let st = unsafe {
        bdf_binary(ctx(), op, dtype_id(&T::get_data_type()), lv.len() as i64, lv.as_ptr(), rv.len() as i64, rv.as_ptr(), outs.as_mut_ptr())
    };
    if st != BDF_OK { return Err(to_arrow_error(st)); }
    Ok(finish::<T>(vals, bits, &outs))
}

/// op: 0 abs, 1 sin, 2 cos, 3 tan, 4 acos, 5 asin, 6 atan, 7 cbrt, 8 ceil, 9 cosh, 10 degrees, 11 exp, 12 expm1,
/// 13 floor, 14 log10, 15 log2, 16 radians, 17 round, 18 sinh, 19 sqrt, 20 tanh (bdf_unop)
pub fn gpu_unary<T: ArrowNumericType>(op: c_int, array: Vec<&PrimitiveArray<T>>) -> Result<Vec<PrimitiveArray<T>>, ArrowError> {
    let v: Vec<BdfView> = array.iter().map(|a| view(*a)).collect();
    let (vals, bits, mut outs) = alloc_outputs::<T>(&array.iter().map(|a| a.len()).collect::<Vec<_>>());
    let st = unsafe { bdf_unary(ctx(), op, dtype_id(&T::get_data_type()), v.len() as i64, v.as_ptr(), outs.as_mut_ptr()) };
    if st != BDF_OK { return Err(to_arrow_error(st)); }
    Ok(finish::<T>(vals, bits, &outs))
}

fn alloc_outputs<T: ArrowPrimitiveType>(lens: &[usize]) -> (Vec<MutableBuffer>, Vec<MutableBuffer>, Vec<BdfOut>) {
    let width = std::mem::size_of::<T::Native>();
    // Both buffers get their FINAL length before the call (zero-filled once, as arrow's own kernels do with `with_bitset`): the
    // library then writes into initialised memory of the right size and nothing has to be resized afterwards -- on arrow
    // versions where `MutableBuffer::resize` zero-fills the grown range, resizing AFTER the call would wipe the results.
    let mut vals: Vec<MutableBuffer> = lens.iter().map(|&n| MutableBuffer::new(n * width).with_bitset(n * width, false)).collect();
    let mut bits: Vec<MutableBuffer> = lens.iter().map(|&n| MutableBuffer::new((n + 7) / 8).with_bitset((n + 7) / 8, false)).collect();
    let outs = (0..lens.len()).map(|i| BdfOut {
        values: vals[i].raw_data_mut() as *mut c_void, validity: bits[i].raw_data_mut(), len: lens[i] as i64, null_count: 0, has_validity: 0,
    }).collect();
    (vals, bits, outs)
}

fn finish<T: ArrowNumericType>(vals: Vec<MutableBuffer>, bits: Vec<MutableBuffer>, outs: &[BdfOut]) -> Vec<PrimitiveArray<T>> {
    outs.iter().zip(vals.into_iter().zip(bits.into_iter())).map(|(o, (v, b))| {
        let len = o.len as usize;   // == the length the buffers were created with (bdf_out.len is checked by the library)
        let nulls = if o.has_validity != 0 { Some(b.freeze()) } else { None };
        let data = ArrayData::new(T::get_data_type(), len, Some(o.null_count as usize), nulls, 0, vec![v.freeze()], vec![]);
        PrimitiveArray::<T>::from(Arc::new(data))
    }).collect()
}

/// coalesce / greatest / least / nanvl (bdf_row_fn 0..3) over columns given as their chunks: scalar.rs's empty stubs with Spark's
/// definitions.  Every column is uploaded, bdf_rowwise_dev runs on them, the result comes back (zip(): the smallest chunk count).
pub fn gpu_rowwise<T: ArrowNumericType>(func: c_int, columns: Vec<Vec<&PrimitiveArray<T>>>) -> Result<Vec<PrimitiveArray<T>>, ArrowError> {
    let dtype = dtype_id(&T::get_data_type());
    let mut cols: Vec<*mut BdfCol> = Vec::new();
    let free = |cols: &Vec<*mut BdfCol>| for c in cols { unsafe { bdf_col_free(ctx(), *c) } };
    for chunks in &columns {
        let v: Vec<BdfView> = chunks.iter().map(|a| view(*a)).collect();
        let mut col: *mut BdfCol = std::ptr::null_mut();
        let st = unsafe { bdf_upload(ctx(), dtype, v.len() as i64, v.as_ptr(), 0, &mut col) };
        if st != BDF_OK { free(&cols); return Err(to_arrow_error(st)); }
        cols.push(col);
    }
    let args: Vec<BdfArg> = cols.iter().map(|c| BdfArg { column: *c as *const BdfCol, bits: 0, valid: 1 }).collect();
    let mut res: *mut BdfCol = std::ptr::null_mut();
    let st = unsafe { bdf_rowwise_dev(ctx(), func, args.len() as i32, args.as_ptr(), &mut res) };
    if st != BDF_OK { free(&cols); return Err(to_arrow_error(st)); }
    let n = columns.iter().map(|c| c.len()).min().unwrap_or(0);
    let (vals, bits, mut outs) = alloc_outputs::<T>(&columns[0][..n].iter().map(|a| a.len()).collect::<Vec<_>>());
    let st = unsafe { bdf_download(ctx(), res, outs.as_mut_ptr()) };
    unsafe { bdf_col_free(ctx(), res) };
    free(&cols);
    if st != BDF_OK { return Err(to_arrow_error(st)); }
    Ok(finish::<T>(vals, bits, &outs))
}

/// Dates and timestamps: the temporal function `func` (bdf_temporal_fn: 0 year .. 6 hour .. 17 to_timestamp) over every chunk of a column
/// whose DataType is Date32 / Date64 / Timestamp / Time32 / Time64; R is the result type bdf_temporal_result reports: Int32Type for the
/// fields, Date32Type for to_date .. next_day, T for date_trunc, Int64Type for unix_timestamp, the Timestamp*Type of the target unit for
/// to_timestamp.  The chunks keep their layout: T::Native and R::Native are the physical i32 / i64.  The arrays carry the DataType the
/// library reports, so a to_timestamp result keeps the input's tz.
pub fn gpu_temporal<T: ArrowPrimitiveType, R: ArrowPrimitiveType>(func: c_int, arg: i64, array: Vec<&PrimitiveArray<T>>)
    -> Result<Vec<PrimitiveArray<R>>, ArrowError>
{
    let mut tz = None;
    let ty = temporal_type(&T::get_data_type(), &mut tz)
        .ok_or_else(|| ArrowError::ComputeError(format!("{:?} is not a date, time or timestamp type", T::get_data_type())))?;
    let mut dt: i32 = -1;
    let mut out_ty = BdfTemporalType { kind: 0, unit: 0, tz: std::ptr::null() };
    let st = unsafe { bdf_temporal_result(func, &ty, arg, &mut dt, &mut out_ty) };
    if st != BDF_OK { return Err(to_arrow_error(st)); }
    let result_type = temporal_data_type(&out_ty).unwrap_or_else(R::get_data_type);
    // R must have the reported physical width and, for a temporal result, the reported kind and unit (the tz comes from the library)
    let mut keep = None;
    let same_kind = match (temporal_type(&R::get_data_type(), &mut keep), out_ty.kind) {
        (None, 0) => true,
        (Some(r), k) => r.kind == k && r.unit == out_ty.unit,
        _ => false,
    };
    if dt != physical_id(&R::get_data_type()) || !same_kind {
        return Err(ArrowError::ComputeError(format!("{:?} is not the result type of temporal function {}: {:?}", R::get_data_type(), func, result_type)));
    }
    let v: Vec<BdfView> = array.iter().map(|a| view(*a)).collect();
    let (vals, bits, mut outs) = alloc_outputs::<R>(&array.iter().map(|a| a.len()).collect::<Vec<_>>());
    let st = unsafe { bdf_temporal(ctx(), func, &ty, arg, v.len() as i64, v.as_ptr(), outs.as_mut_ptr()) };
    if st != BDF_OK { return Err(to_arrow_error(st)); }
    Ok(finish_as::<R>(vals, bits, &outs, &result_type))
}

/// The bdf_dtype of a primitive DataType: numeric types by dtype_id, temporal types by their physical width (Date32 / Time32: Int32).
fn physical_id(t: &DataType) -> c_int {
    let mut keep = None;
    match temporal_type(t, &mut keep) {
        Some(tt) => if tt.kind == 1 || tt.kind == 4 { 2 } else { 3 },
        None => dtype_id(t),
    }
}

/// The arrow DataType of a bdf_temporal_type (None for kind 0).
fn temporal_data_type(t: &BdfTemporalType) -> Option<DataType> {
    let unit = match t.unit { 0 => TimeUnit::Second, 1 => TimeUnit::Millisecond, 2 => TimeUnit::Microsecond, _ => TimeUnit::Nanosecond };
    match t.kind {
        1 => Some(DataType::Date32(DateUnit::Day)),
        2 => Some(DataType::Date64(DateUnit::Millisecond)),
        3 => {
            let tz = if t.tz.is_null() { None } else { Some(unsafe { std::ffi::CStr::from_ptr(t.tz) }.to_string_lossy().into_owned()) };
            Some(DataType::Timestamp(unit, tz.map(Arc::new)))
        }
        4 => Some(DataType::Time32(unit)),
        5 => Some(DataType::Time64(unit)),
        _ => None,
    }
}

fn finish_as<R: ArrowPrimitiveType>(vals: Vec<MutableBuffer>, bits: Vec<MutableBuffer>, outs: &[BdfOut], data_type: &DataType) -> Vec<PrimitiveArray<R>> {
    outs.iter().zip(vals.into_iter().zip(bits.into_iter())).map(|(o, (v, b))| {
        let nulls = if o.has_validity != 0 { Some(b.freeze()) } else { None };
        let data = ArrayData::new(data_type.clone(), o.len as usize, Some(o.null_count as usize), nulls, 0, vec![v.freeze()], vec![]);
        PrimitiveArray::<R>::from(Arc::new(data))
    }).collect()
}

// In src/functions/scalar.rs the bodies become:
//   pub fn add<T>(left, right)          -> gpu_binary(0, left, right)     // was: left.par_iter().zip(..).map(compute::add)   (scalar.rs:16-32)
//   pub fn subtract<T>(left, right)     -> gpu_binary(1, left, right)     // (scalar.rs:34-50)
//   pub fn divide<T>(left, right)       -> gpu_binary(3, left, right)     // Err(ArrowError::DivideByZero) preserved (scalar.rs:51-68)
//   pub fn multiply / par_multiply<T>   -> gpu_binary(2, left, right)     // (scalar.rs:69-103)
//   pub fn abs/sin/cos/tan/acos/...<T>  -> gpu_unary(op, array)           // was: scalar_op(a, |a| Ok(num::Float::sin(a)))      (scalar.rs:106-457)
//   pub fn coalesce / greatest / least<T>(arrays: Vec<Vec<&PrimitiveArray<T>>>) -> gpu_rowwise(0 | 1 | 2, arrays)   // stubs (scalar.rs:180,264,286)
//   pub fn nanv1<T>(a, b)               -> gpu_rowwise(3, vec![a, b])     // Spark's nanvl (stub, scalar.rs:343)
//   pub fn hour<T>(array) -> Result<Vec<Int32Array>>  -> gpu_temporal::<T, Int32Type>(6, 0, array)   // was: compute::hour per chunk (scalar.rs:267-273)
//   the stubs: year 0, quarter 1, month 2, day_of_month 3, day_of_year 4, day_of_week 5, minute 7, second 8  -> gpu_temporal::<T, Int32Type>
//              to_date 9, date_add 10 (arg days), date_sub 11, add_months 12 (arg months), last_day 13, next_day 14 (arg 1..7)
//                                                                   -> gpu_temporal::<T, Date32Type>
//              date_trunc 15 (arg bdf_trunc_unit) -> gpu_temporal::<T, T>; unix_timestamp 16 -> Int64Type; to_timestamp 17 -> Timestamp*Type
