//! Replacement bodies for src/functions/array.rs (ArrayFunctions; signatures unchanged) and the size / explode stubs of
//! src/functions/scalar.rs.  UNCOMPILED here -- see ../README.md.  Rules and departures: include/b200df.h "list columns".
use std::os::raw::c_void;

use arrow::array::{Array, ArrayData, BooleanArray, Int32Array, ListArray, PrimitiveArray, UInt32Array};
use arrow::buffer::MutableBuffer;
use arrow::datatypes::{ArrowNumericType, DataType, ToByteSlice};
use arrow::error::ArrowError;

use crate::ffi::*;

/// A bdf_list_view of a ListArray: its offsets and validity from the list's offset, the child as a bdf_view (its own offset applies).
pub fn list_view<T: ArrowNumericType>(a: &ListArray) -> BdfListView {
    let data = a.data();
    let values = a.values();
    let child = values.as_any().downcast_ref::<PrimitiveArray<T>>().expect("a List of T");
    BdfListView {
        offsets: data.buffers()[0].raw_data() as *const i32,
        validity: data.null_bitmap().as_ref().map_or(std::ptr::null(), |b| b.bits.raw_data()),
        len: a.len() as i64,
        offset: a.offset() as i64,
        null_count: a.null_count() as i64,
        values: view(child),
    }
}

/// T::Native in the low bytes of a u64 (the search value of bdf_list_find_dev / BDF_LIST_REMOVE).
pub fn bits_of<T: ArrowNumericType>(v: T::Native) -> u64 {
    let mut out = 0u64;
    let b = [v].to_byte_slice();
    unsafe { std::ptr::copy_nonoverlapping(b.as_ptr(), &mut out as *mut u64 as *mut u8, b.len()) };
    out
}

fn check(st: i32) -> Result<(), ArrowError> {
    match st {
        BDF_OK => Ok(()),
        BDF_LENGTH_MISMATCH => Err(ArrowError::ComputeError("Expected array a and b to have the same length".to_string())),
        BDF_WOULD_PANIC => panic!("called `Option::unwrap()` on a `None` value"),   // array_max / array_min of an empty list
        st => Err(to_arrow_error(st)),
    }
}

fn upload<T: ArrowNumericType>(a: &ListArray) -> Result<*mut BdfList, ArrowError> {
    let v = list_view::<T>(a);
    let mut l = std::ptr::null_mut();
    check(unsafe { bdf_list_upload(ctx_one_gpu(), dtype_id(&T::get_data_type()), 1, &v, 0, &mut l) })?;
    Ok(l)
}

/// A one-chunk device list -> ListArray (offsets, validity, child values and validity downloaded into MutableBuffers).
fn download_list<T: ArrowNumericType>(l: *mut BdfList) -> Result<ListArray, ArrowError> {
    let (mut len, mut nulls, mut n) = (0i64, 0i64, 0i64);
    check(unsafe { bdf_list_chunk_info(ctx_one_gpu(), l, 0, &mut len, &mut nulls, &mut n) })?;
    let w = std::mem::size_of::<T::Native>();
    let mut off = MutableBuffer::new((len as usize + 1) * 4).with_bitset((len as usize + 1) * 4, false);
    let mut val = MutableBuffer::new(len as usize / 8 + 1).with_bitset(len as usize / 8 + 1, false);
    let mut vals = MutableBuffer::new(n as usize * w).with_bitset(n as usize * w, false);
    let mut vval = MutableBuffer::new(n as usize / 8 + 1).with_bitset(n as usize / 8 + 1, false);
    let mut out = BdfListOut {
        offsets: off.raw_data_mut() as *mut i32, validity: val.raw_data_mut(), values: vals.raw_data_mut() as *mut c_void,
        value_validity: vval.raw_data_mut(), null_count: 0, value_null_count: 0, has_validity: 0, has_value_validity: 0,
    };
    check(unsafe { bdf_list_download(ctx_one_gpu(), l, &mut out) })?;
    unsafe { bdf_list_free(ctx_one_gpu(), l) };
    let mut child = ArrayData::builder(T::get_data_type()).len(n as usize).add_buffer(vals.freeze());
    if out.has_value_validity != 0 { child = child.null_bit_buffer(vval.freeze()); }
    let mut list = ArrayData::builder(DataType::List(Box::new(T::get_data_type()))).len(len as usize).add_buffer(off.freeze())
        .add_child_data(child.build());
    if out.has_validity != 0 { list = list.null_bit_buffer(val.freeze()); }
    Ok(ListArray::from(list.build()))
}

fn download_col<A: From<ArrayData>>(dtype: DataType, col: *mut BdfCol) -> Result<A, ArrowError> {
    let (mut len, mut nulls, mut hv) = (0i64, 0i64, 0i32);
    check(unsafe { bdf_col_chunk_info(ctx_one_gpu(), col, 0, &mut len, &mut nulls, &mut hv) })?;
    let bytes = if dtype == DataType::Boolean { len as usize / 8 + 1 } else { len as usize * 8 };
    let mut vals = MutableBuffer::new(bytes).with_bitset(bytes, false);
    let mut bits = MutableBuffer::new(len as usize / 8 + 1).with_bitset(len as usize / 8 + 1, false);
    let mut o = BdfOut { values: vals.raw_data_mut() as *mut c_void, validity: bits.raw_data_mut(), len, null_count: 0, has_validity: 0 };
    check(unsafe { bdf_download(ctx_one_gpu(), col, &mut o) })?;
    unsafe { bdf_col_free(ctx_one_gpu(), col) };
    let mut b = ArrayData::builder(dtype).len(len as usize).add_buffer(vals.freeze());
    if o.has_validity != 0 { b = b.null_bit_buffer(bits.freeze()); }
    Ok(A::from(b.build()))
}

fn find<T: ArrowNumericType>(f: i32, a: &ListArray, v: T::Native) -> Result<*mut BdfCol, ArrowError> {
    let l = upload::<T>(a)?;
    let mut out = std::ptr::null_mut();
    let st = unsafe { bdf_list_find_dev(ctx_one_gpu(), f, l, bits_of::<T>(v), &mut out) };
    unsafe { bdf_list_free(ctx_one_gpu(), l) };
    check(st)?;
    Ok(out)
}

pub fn array_contains<T: ArrowNumericType>(a: &ListArray, v: T::Native) -> Result<BooleanArray, ArrowError> {
    download_col(DataType::Boolean, find::<T>(BDF_LIST_CONTAINS, a, v)?)
}

pub fn array_position<T: ArrowNumericType>(a: &ListArray, v: T::Native) -> Result<Int32Array, ArrowError> {
    download_col(DataType::Int32, find::<T>(BDF_LIST_POSITION, a, v)?)
}

fn reduce<T: ArrowNumericType, A: From<ArrayData>>(f: i32, a: &ListArray, dtype: DataType) -> Result<A, ArrowError> {
    let l = upload::<T>(a)?;
    let mut out = std::ptr::null_mut();
    let st = unsafe { bdf_list_reduce_dev(ctx_one_gpu(), f, l, &mut out) };
    unsafe { bdf_list_free(ctx_one_gpu(), l) };
    check(st)?;
    download_col(dtype, out)
}

pub fn array_max<T: ArrowNumericType>(a: &ListArray) -> Result<PrimitiveArray<T>, ArrowError> { reduce::<T, _>(BDF_LIST_MAX, a, T::get_data_type()) }
pub fn array_min<T: ArrowNumericType>(a: &ListArray) -> Result<PrimitiveArray<T>, ArrowError> { reduce::<T, _>(BDF_LIST_MIN, a, T::get_data_type()) }
pub fn size<T: ArrowNumericType>(a: &ListArray) -> Result<Int32Array, ArrowError> { reduce::<T, _>(BDF_LIST_SIZE, a, DataType::Int32) }

fn transform<T: ArrowNumericType>(f: i32, a: &ListArray, v: T::Native, count: i64) -> Result<ListArray, ArrowError> {
    let l = upload::<T>(a)?;
    let mut out = std::ptr::null_mut();
    let st = unsafe { bdf_list_transform_dev(ctx_one_gpu(), f, l, bits_of::<T>(v), count, &mut out) };
    unsafe { bdf_list_free(ctx_one_gpu(), l) };
    check(st)?;
    download_list::<T>(out)
}

pub fn array_remove<T: ArrowNumericType>(a: &ListArray, v: T::Native) -> Result<ListArray, ArrowError> { transform::<T>(BDF_LIST_REMOVE, a, v, 0) }
pub fn array_sort<T: ArrowNumericType>(a: &ListArray) -> Result<ListArray, ArrowError> { transform::<T>(BDF_LIST_SORT, a, T::default_value(), 0) }
pub fn array_distinct<T: ArrowNumericType>(a: &ListArray) -> Result<ListArray, ArrowError> { transform::<T>(BDF_LIST_DISTINCT, a, T::default_value(), 0) }
pub fn array_repeat<T: ArrowNumericType>(a: &ListArray, count: i32) -> Result<ListArray, ArrowError> {
    transform::<T>(BDF_LIST_REPEAT, a, T::default_value(), count as i64)
}

fn set<T: ArrowNumericType>(f: i32, a: &ListArray, b: &ListArray) -> Result<ListArray, ArrowError> {
    let la = upload::<T>(a)?;
    let lb = upload::<T>(b)?;
    let mut out = std::ptr::null_mut();
    let st = unsafe { bdf_list_set_dev(ctx_one_gpu(), f, la, lb, &mut out) };
    unsafe { bdf_list_free(ctx_one_gpu(), la); bdf_list_free(ctx_one_gpu(), lb) };
    check(st)?;
    download_list::<T>(out)
}

pub fn array_except<T: ArrowNumericType>(a: &ListArray, b: &ListArray) -> Result<ListArray, ArrowError> { set::<T>(BDF_LIST_EXCEPT, a, b) }
pub fn array_intersect<T: ArrowNumericType>(a: &ListArray, b: &ListArray) -> Result<ListArray, ArrowError> { set::<T>(BDF_LIST_INTERSECT, a, b) }
pub fn array_union<T: ArrowNumericType>(a: &ListArray, b: &ListArray) -> Result<ListArray, ArrowError> { set::<T>(BDF_LIST_UNION, a, b) }

/// (parent row numbers, values): one row per element of every valid list; take other columns with the row numbers.
pub fn explode<T: ArrowNumericType>(a: &ListArray) -> Result<(UInt32Array, PrimitiveArray<T>), ArrowError> {
    let l = upload::<T>(a)?;
    let (mut rows, mut vals) = (std::ptr::null_mut(), std::ptr::null_mut());
    let st = unsafe { bdf_list_explode_dev(ctx_one_gpu(), l, &mut rows, &mut vals) };
    unsafe { bdf_list_free(ctx_one_gpu(), l) };
    check(st)?;
    Ok((download_col(DataType::UInt32, rows)?, download_col(T::get_data_type(), vals)?))
}

/// Column::take of a ListArray column (DataFrame::sort / join / limit dispatch here for DataType::List): out[i] = a[indices[i]], a
/// null index gives a null list; an index past the end is an error.  `indices` is a device UInt32 column (the sort's or the join's).
pub fn take<T: ArrowNumericType>(a: &ListArray, indices: *const BdfCol) -> Result<ListArray, ArrowError> {
    let l = upload::<T>(a)?;
    let mut out = std::ptr::null_mut();
    let st = unsafe { bdf_list_take_dev(ctx_one_gpu(), l, indices, &mut out) };
    unsafe { bdf_list_free(ctx_one_gpu(), l) };
    check(st)?;
    download_list::<T>(out)
}

/// ChunkedArray::filter of a ListArray chunk: the lists where the device Boolean mask is valid and true.
pub fn filter<T: ArrowNumericType>(a: &ListArray, mask: *const BdfCol) -> Result<ListArray, ArrowError> {
    let l = upload::<T>(a)?;
    let mut out = std::ptr::null_mut();
    let st = unsafe { bdf_list_filter_dev(ctx_one_gpu(), l, mask, &mut out) };
    unsafe { bdf_list_free(ctx_one_gpu(), l) };
    check(st)?;
    download_list::<T>(out)
}

/// ArrayFunction::CollectList / CollectSet per group of the device key columns: (key columns, one list per group).  collect_list: the
/// valid values in row order; collect_set: the distinct valid values ascending (NaN greatest, -0.0 == 0.0).  Never a null list.
fn collect<T: ArrowNumericType>(f: i32, keys: &[*const BdfCol], x: *const BdfCol) -> Result<(Vec<*mut BdfCol>, ListArray), ArrowError> {
    let agg = BdfGroupAgg { column: x, function: f };
    let mut out_keys = vec![std::ptr::null_mut(); keys.len()];
    let (mut out, mut list, mut n_groups) = (std::ptr::null_mut(), std::ptr::null_mut(), 0i64);
    check(unsafe { bdf_group_by_lists_dev(ctx_one_gpu(), keys.len() as i32, keys.as_ptr(), 1, &agg, out_keys.as_mut_ptr(), &mut out, &mut list,
                                          &mut n_groups) })?;
    Ok((out_keys, download_list::<T>(list)?))
}

pub fn collect_list<T: ArrowNumericType>(keys: &[*const BdfCol], x: *const BdfCol) -> Result<(Vec<*mut BdfCol>, ListArray), ArrowError> {
    collect::<T>(BDF_GROUP_COLLECT_LIST, keys, x)
}

pub fn collect_set<T: ArrowNumericType>(keys: &[*const BdfCol], x: *const BdfCol) -> Result<(Vec<*mut BdfCol>, ListArray), ArrowError> {
    collect::<T>(BDF_GROUP_COLLECT_SET, keys, x)
}

// In src/functions/array.rs (ArrayFunctions):
//   pub fn array_contains<T>(array, val)  -> array_gpu::array_contains::<T>(array, val)
//   pub fn array_position<T>(array, val)  -> array_gpu::array_position::<T>(array, val)
//   pub fn array_remove / array_max / array_min / array_repeat / array_except / array_intersect / array_union  -> the same names
//   fn array_sort / array_distinct (private)                                                                 -> the same names
