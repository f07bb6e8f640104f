//! Device-resident frames: how `DataFrame::{from_arrow, to_arrow, sort}`, the group-by aggregate and a fused run of Calculations map onto
//! libb200df.so.  UNCOMPILED here (see ../README.md); the same flow is exercised from Python in
//! rust-dataframe_b200/frame.py (tests/test_frame.py, tests/test_ipc.py, tests/test_sort_gpu.py).
use std::ffi::{CStr, CString};
use std::os::raw::c_char;

use crate::ffi::*;

/// Columns of a frame that live in HBM: one `BdfCol` per numeric/boolean column, one chunk per RecordBatch.
pub struct DeviceColumns {
    pub names: Vec<String>,
    pub cols: Vec<*mut BdfCol>,
}

impl Drop for DeviceColumns {
    fn drop(&mut self) {
        for c in &self.cols {
            if !c.is_null() { unsafe { bdf_col_free(dev(), *c) }; }
        }
    }
}

/// The frames of this module live on ONE GPU: sort, take and the IPC readers are one-GPU entries (include/b200df.h).
fn dev() -> *mut BdfCtx { ctx_one_gpu() }

/// DataFrame::from_arrow (src/dataframe.rs:391-407) for the columns on the path: the file is mapped and its body buffers
/// go straight to the device.  Columns reported with dtype -1 (Utf8, List, ...) keep coming from arrow's FileReader.
pub fn from_arrow_device(path: &str) -> Result<DeviceColumns, String> {
    let cpath = CString::new(path).unwrap();
    let mut f: *mut BdfIpc = std::ptr::null_mut();
    check(unsafe { bdf_ipc_open(cpath.as_ptr(), &mut f) })?;
    // the file handle is closed on every path out of this function
    struct Close(*mut BdfIpc);
    impl Drop for Close { fn drop(&mut self) { unsafe { bdf_ipc_close(self.0) } } }
    let _close = Close(f);
    let (mut n_cols, mut n_batches, mut n_rows) = (0i32, 0i64, 0i64);
    check(unsafe { bdf_ipc_describe(f, &mut n_cols, &mut n_batches, &mut n_rows) })?;
    let mut wanted = vec![];
    let mut names = vec![];
    for c in 0..n_cols {
        let (mut name, mut dtype, mut nullable): (*const c_char, i32, i32) = (std::ptr::null(), -1, 0);
        check(unsafe { bdf_ipc_column(f, c, &mut name, &mut dtype, &mut nullable) })?;
        if dtype >= 0 {
            wanted.push(c);
            names.push(unsafe { CStr::from_ptr(name) }.to_string_lossy().into_owned());
        }
    }
    if wanted.is_empty() {
        return Ok(DeviceColumns { names, cols: vec![] });   // no numeric/boolean column: nothing for the device (bdf_ipc_read rejects n_cols == 0)
    }
    let mut cols = vec![std::ptr::null_mut(); wanted.len()];
    check(unsafe { bdf_ipc_read(dev(), f, wanted.len() as i32, wanted.as_ptr(), 0, cols.as_mut_ptr()) })?;   // synchronous: the copies are done
    Ok(DeviceColumns { names, cols })
}

/// DataFrame::to_arrow (src/dataframe.rs:515-525): chunk b of every column is RecordBatch b.
pub fn to_arrow_device(frame: &DeviceColumns, path: &str) -> Result<(), String> {
    let cpath = CString::new(path).unwrap();
    let cnames: Vec<CString> = frame.names.iter().map(|s| CString::new(s.as_str()).unwrap()).collect();
    let name_ptrs: Vec<*const c_char> = cnames.iter().map(|s| s.as_ptr()).collect();
    let col_ptrs: Vec<*const BdfCol> = frame.cols.iter().map(|c| *c as *const BdfCol).collect();
    check(unsafe { bdf_ipc_write(dev(), cpath.as_ptr(), col_ptrs.len() as i32, name_ptrs.as_ptr(), col_ptrs.as_ptr()) })
}

/// DataFrame::sort (src/dataframe.rs:194-222): criteria = (column index, descending); nulls last like the reference.
pub fn sort_device(frame: &DeviceColumns, criteria: &[(usize, bool)]) -> Result<DeviceColumns, String> {
    if criteria.is_empty() {
        return Err("Sort criteria cannot be empty".to_string());
    }
    let keys: Vec<BdfSortKey> = criteria.iter().map(|(c, d)| BdfSortKey { column: frame.cols[*c], descending: *d as i32 }).collect();
    let mut indices: *mut BdfCol = std::ptr::null_mut();
    check(unsafe { bdf_sort_indices_dev(dev(), keys.len() as i32, keys.as_ptr(), &mut indices) })?;   // lexsort_to_indices
    // both the index column and the columns taken so far are owned by guards: an error half-way frees them (raw pointers have no Drop)
    let idx = DeviceColumns { names: vec![], cols: vec![indices] };
    let mut out = DeviceColumns { names: frame.names.clone(), cols: Vec::with_capacity(frame.cols.len()) };
    for c in &frame.cols {
        let mut taken: *mut BdfCol = std::ptr::null_mut();
        check(unsafe { bdf_take_dev(dev(), *c, idx.cols[0], &mut taken) })?;                            // sort_by_indices -> Column::take
        out.cols.push(taken);
    }
    Ok(out)
}

/// DataFrame::sort followed by DataFrame::limit(k) as one call: the first k rows of the sort, chosen on the device without sorting every
/// row (bdf_top_k_indices_dev), then every column taken at them.  A negative k gives no rows, as limit does.
pub fn top_k_device(frame: &DeviceColumns, criteria: &[(usize, bool)], k: i64) -> Result<DeviceColumns, String> {
    if criteria.is_empty() {
        return Err("Sort criteria cannot be empty".to_string());
    }
    let keys: Vec<BdfSortKey> = criteria.iter().map(|(c, d)| BdfSortKey { column: frame.cols[*c], descending: *d as i32 }).collect();
    let mut indices: *mut BdfCol = std::ptr::null_mut();
    check(unsafe { bdf_top_k_indices_dev(dev(), keys.len() as i32, keys.as_ptr(), k.max(0), &mut indices) })?;
    let idx = DeviceColumns { names: vec![], cols: vec![indices] };
    let mut out = DeviceColumns { names: frame.names.clone(), cols: Vec::with_capacity(frame.cols.len()) };
    for c in &frame.cols {
        let mut taken: *mut BdfCol = std::ptr::null_mut();
        check(unsafe { bdf_take_dev(dev(), *c, idx.cols[0], &mut taken) })?;
        out.cols.push(taken);
    }
    Ok(out)
}

/// Column::take of one column of a frame, as sort / join / limit call it: a DataType::List column goes through bdf_list_take_dev (whole
/// lists, one chunk; a null index gives a null list), every other column through bdf_take_dev.  ChunkedArray::filter dispatches the same
/// way to bdf_list_filter_dev, which keeps the chunks, so list chunk b stays RecordBatch b for to_arrow (bdf_ipc_write_lists).
pub enum DeviceColumn { Flat(*mut BdfCol), List(*mut BdfList) }

pub fn take_column(c: &DeviceColumn, indices: *const BdfCol) -> Result<DeviceColumn, String> {
    match c {
        DeviceColumn::Flat(col) => {
            let mut out: *mut BdfCol = std::ptr::null_mut();
            check(unsafe { bdf_take_dev(dev(), *col, indices, &mut out) })?;
            Ok(DeviceColumn::Flat(out))
        }
        DeviceColumn::List(list) => {
            let mut out: *mut BdfList = std::ptr::null_mut();
            check(unsafe { bdf_list_take_dev(dev(), *list, indices, &mut out) })?;
            Ok(DeviceColumn::List(out))
        }
    }
}

pub fn filter_column(c: &DeviceColumn, mask: *const BdfCol) -> Result<DeviceColumn, String> {
    match c {
        DeviceColumn::Flat(col) => {
            let mut out: *mut BdfCol = std::ptr::null_mut();
            check(unsafe { bdf_filter_dev(dev(), *col, mask, &mut out) })?;
            Ok(DeviceColumn::Flat(out))
        }
        DeviceColumn::List(list) => {
            let mut out: *mut BdfList = std::ptr::null_mut();
            check(unsafe { bdf_list_filter_dev(dev(), *list, mask, &mut out) })?;
            Ok(DeviceColumn::List(out))
        }
    }
}

/// One aggregate of the plan `Dataset::try_aggregate` makes (src/expression.rs:114-221): the ones on this path.
#[derive(Clone, Copy, PartialEq)]
pub enum GroupFn { Sum, Count, Min, Max }

/// `Transformation::GroupAggregate` (a `panic!("aggregations not supported")` in src/evaluation.rs:73): group by ONE key column,
/// output = the key column, then `sum(x)` / `min(x)` / `max(x)` (type of x) or `count(x)` (UInt32) per requested aggregate -- the
/// names and types of the planned schema.  Groups in ascending key order, the null key last.
pub fn group_aggregate_device(frame: &DeviceColumns, key: usize, aggr: &[(usize, GroupFn)]) -> Result<DeviceColumns, String> {
    const BDF_U32: i32 = 6;   // include/b200df.h bdf_dtype
    let mut value_cols: Vec<usize> = vec![];
    for (c, _) in aggr { if !value_cols.contains(c) { value_cols.push(*c); } }
    let vals: Vec<*const BdfCol> = value_cols.iter().map(|c| frame.cols[*c] as *const BdfCol).collect();
    let mut keys: *mut BdfCol = std::ptr::null_mut();
    let mut n_groups = 0i64;
    let null = std::ptr::null_mut();
    let mut outs = vec![BdfGroupOut { sum: null, count: null, min: null, max: null }; vals.len()];
    check(unsafe { bdf_group_aggregate_dev(dev(), frame.cols[key], vals.len() as i32, vals.as_ptr(), &mut keys, outs.as_mut_ptr(), &mut n_groups) })?;
    // every column the library returned is owned by a guard from here on: the ones the plan did not ask for are dropped with it
    let mut spare = DeviceColumns { names: vec![], cols: outs.iter().flat_map(|o| vec![o.sum, o.count, o.min, o.max]).collect() };
    let mut out = DeviceColumns { names: vec![frame.names[key].clone()], cols: vec![keys] };
    for (c, f) in aggr {
        let j = value_cols.iter().position(|v| v == c).unwrap();
        let slot = 4 * j + match f { GroupFn::Sum => 0, GroupFn::Count => 1, GroupFn::Min => 2, GroupFn::Max => 3 };
        let col = spare.cols[slot];
        if col.is_null() {
            return Err("min/max need T::Native: Ord (integer columns), or the aggregate was requested twice".to_string());
        }
        let x = &frame.names[*c];
        match f {
            GroupFn::Count => {   // count(x) is planned as UInt32; group sizes are below 2^32 (row numbers are UInt32), the cast cannot fail
                let mut c32: *mut BdfCol = std::ptr::null_mut();
                check(unsafe { bdf_cast_dev(dev(), BDF_U32, col, &mut c32) })?;
                out.names.push(format!("count({})", x));
                out.cols.push(c32);
            }
            _ => {
                spare.cols[slot] = null;   // moves to the result
                out.names.push(format!("{}({})", match f { GroupFn::Sum => "sum", GroupFn::Min => "min", _ => "max" }, x));
                out.cols.push(col);
            }
        }
    }
    Ok(out)
}

/// Every function `Dataset::try_aggregate` plans and the device computes (AggregateFunction order); Kurtosis, Skewness, StdDev,
/// SumDistinct and Variance are refused by the plan itself ("Aggregation not yet supported").
#[derive(Clone, Copy, PartialEq)]
pub enum GroupByFn { Sum, Max, Min, Avg, Count, CountDistinct, First, Last }

/// `Transformation::GroupAggregate(groups, aggr)` over any number of key columns: output = the key columns, then `fn(x)` per
/// (column, function) of the flattened aggregations -- `count(x)` / `count_distinct(x)` cast to the planned UInt32, `avg(x)` kept
/// Float64, the others of x's type.  Groups in the order DataFrame::sort gives the keys (ascending, nulls last per key).
pub fn group_by_device(frame: &DeviceColumns, keys: &[usize], aggr: &[(usize, GroupByFn)]) -> Result<DeviceColumns, String> {
    const BDF_U32: i32 = 6;   // include/b200df.h bdf_dtype
    let key_cols: Vec<*const BdfCol> = keys.iter().map(|k| frame.cols[*k] as *const BdfCol).collect();
    let pairs: Vec<BdfGroupAgg> = aggr.iter().map(|(c, f)| BdfGroupAgg { column: frame.cols[*c], function: *f as i32 }).collect();
    let mut out_keys = vec![std::ptr::null_mut(); key_cols.len()];
    let mut out = vec![std::ptr::null_mut(); pairs.len()];
    let mut n_groups = 0i64;
    check(unsafe { bdf_group_by_dev(dev(), key_cols.len() as i32, key_cols.as_ptr(), pairs.len() as i32, pairs.as_ptr(), out_keys.as_mut_ptr(),
                                    out.as_mut_ptr(), &mut n_groups) })?;
    // every returned column is owned by `res` from here on: an early return frees all of them
    let mut res = DeviceColumns { names: keys.iter().map(|k| frame.names[*k].clone()).collect(), cols: out_keys };
    for ((c, f), col) in aggr.iter().zip(out) {
        let name = match f {
            GroupByFn::Sum => "sum", GroupByFn::Max => "max", GroupByFn::Min => "min", GroupByFn::Avg => "avg", GroupByFn::Count => "count",
            GroupByFn::CountDistinct => "count_distinct", GroupByFn::First => "first", GroupByFn::Last => "last",
        };
        res.names.push(format!("{}({})", name, frame.names[*c]));
        res.cols.push(col);
    }
    for (j, (_, f)) in aggr.iter().enumerate() {
        if matches!(f, GroupByFn::Count | GroupByFn::CountDistinct) {   // Int64 -> the planned UInt32 (a group has < 2^32 rows)
            let slot = keys.len() + j;
            let mut c32: *mut BdfCol = std::ptr::null_mut();
            check(unsafe { bdf_cast_dev(dev(), BDF_U32, res.cols[slot], &mut c32) })?;
            unsafe { bdf_col_free(dev(), res.cols[slot]) };
            res.cols[slot] = c32;
        }
    }
    Ok(res)
}

/// `DataFrame::join` (src/dataframe.rs:626-719) with the body of `calc_equijoin_indices` as one call.  `criteria`: (left column,
/// right column) pairs; `join_type`: JoinType's discriminant (Left, Right, Inner, Full -- bdf_join_type).  Output = every column of
/// `left`, then every column of `right`, taken by the index pairs (NULL index -> NULL slot); a name present on both sides becomes
/// `a.<name>` / `b.<name>`, the schema `Dataset::try_join` plans.  Pair order and the departures from the reference: include/b200df.h.
/// BDF_JOIN_LEFT_SEMI / BDF_JOIN_LEFT_ANTI: the columns of `left` only, names unchanged, at the left rows that have (lack) a partner.
pub fn join_device(left: &DeviceColumns, right: &DeviceColumns, criteria: &[(usize, usize)], join_type: i32) -> Result<DeviceColumns, String> {
    let lk: Vec<*const BdfCol> = criteria.iter().map(|(l, _)| left.cols[*l] as *const BdfCol).collect();
    let rk: Vec<*const BdfCol> = criteria.iter().map(|(_, r)| right.cols[*r] as *const BdfCol).collect();
    let (mut li, mut ri, mut n_rows) = (std::ptr::null_mut(), std::ptr::null_mut(), 0i64);
    check(unsafe { bdf_join_indices_dev(dev(), join_type, lk.len() as i32, lk.as_ptr(), rk.as_ptr(), &mut li, &mut ri, &mut n_rows) })?;
    let idx = DeviceColumns { names: vec![], cols: vec![li, ri] };   // freed when this function returns, early or not
    if join_type == BDF_JOIN_LEFT_SEMI || join_type == BDF_JOIN_LEFT_ANTI {
        let mut out = DeviceColumns { names: left.names.clone(), cols: Vec::with_capacity(left.cols.len()) };
        for col in &left.cols {
            let mut taken: *mut BdfCol = std::ptr::null_mut();
            check(unsafe { bdf_take_dev(dev(), *col, idx.cols[0], &mut taken) })?;
            out.cols.push(taken);
        }
        return Ok(out);
    }
    let mut out = DeviceColumns { names: vec![], cols: vec![] };
    for (side, other, prefix, indices) in [(left, right, "a", idx.cols[0]), (right, left, "b", idx.cols[1])] {
        for (name, col) in side.names.iter().zip(&side.cols) {
            let mut taken: *mut BdfCol = std::ptr::null_mut();
            check(unsafe { bdf_take_dev(dev(), *col, indices, &mut taken) })?;
            out.names.push(if other.names.contains(name) { format!("{}.{}", prefix, name) } else { name.clone() });
            out.cols.push(taken);
        }
    }
    Ok(out)
}

/// An as-of join (pandas' merge_asof; include/b200df.h "as-of join"): for every row of `left`, in its order, the row of `right` whose
/// `on.1` key is the last at or before its `on.0` key (BDF_ASOF_BACKWARD), the first at or after it (FORWARD) or the nearer (NEAREST),
/// among the rows whose `by` pairs are equal.  Returns the columns of `right` only, taken by that row (NULL where there is none), one
/// chunk each in `left`'s row order; a name `left` also has becomes `b.<name>` (the caller renames its own column to `a.<name>`, the
/// schema `Dataset::try_join` plans), so the left columns are never copied.
pub fn join_asof_device(left: &DeviceColumns, right: &DeviceColumns, on: (usize, usize), by: &[(usize, usize)], spec: &BdfAsofSpec)
                        -> Result<DeviceColumns, String> {
    let lb: Vec<*const BdfCol> = by.iter().map(|(l, _)| left.cols[*l] as *const BdfCol).collect();
    let rb: Vec<*const BdfCol> = by.iter().map(|(_, r)| right.cols[*r] as *const BdfCol).collect();
    let mut ri: *mut BdfCol = std::ptr::null_mut();
    check(unsafe { bdf_join_asof_dev(dev(), left.cols[on.0], right.cols[on.1], lb.len() as i32, lb.as_ptr(), rb.as_ptr(), spec, &mut ri) })?;
    let idx = DeviceColumns { names: vec![], cols: vec![ri] };   // freed when this function returns, early or not
    let mut out = DeviceColumns { names: vec![], cols: Vec::with_capacity(right.cols.len()) };
    for (name, col) in right.names.iter().zip(&right.cols) {
        let mut taken: *mut BdfCol = std::ptr::null_mut();
        check(unsafe { bdf_take_dev(dev(), *col, idx.cols[0], &mut taken) })?;
        out.names.push(if left.names.contains(name) { format!("b.{}", name) } else { name.clone() });
        out.cols.push(taken);
    }
    Ok(out)
}

/// pandas' `duplicated` over the columns `keys` of `frame` (include/b200df.h "distinct rows and set operations"): a Boolean mask
/// without nulls, chunked like the frame, true for the rows `keep` (BDF_KEEP_FIRST / _LAST / _NONE) marks.  Filter every column with
/// its NOT for `drop_duplicates`.  Not in the reference.
pub fn duplicated_device(frame: &DeviceColumns, keys: &[usize], keep: i32) -> Result<*mut BdfCol, String> {
    let ks: Vec<*const BdfCol> = keys.iter().map(|k| frame.cols[*k] as *const BdfCol).collect();
    let mut mask: *mut BdfCol = std::ptr::null_mut();
    check(unsafe { bdf_duplicated_dev(dev(), ks.len() as i32, ks.as_ptr(), keep, &mut mask) })?;
    Ok(mask)
}

/// Spark's `intersect` / `intersectAll` / `subtract` / `exceptAll` (`op`: BDF_SETOP_*), every column compared by position: the mask
/// of the `left` rows kept, chunked like `left`, in its row order.  Not in the reference.
pub fn set_op_device(left: &DeviceColumns, right: &DeviceColumns, op: i32) -> Result<*mut BdfCol, String> {
    if left.cols.len() != right.cols.len() {
        return Err("Union can only be performed on tables with compatible column types".to_string());
    }
    let lk: Vec<*const BdfCol> = left.cols.iter().map(|c| *c as *const BdfCol).collect();
    let rk: Vec<*const BdfCol> = right.cols.iter().map(|c| *c as *const BdfCol).collect();
    let mut mask: *mut BdfCol = std::ptr::null_mut();
    check(unsafe { bdf_set_op_dev(dev(), op, lk.len() as i32, lk.as_ptr(), rk.as_ptr(), &mut mask) })?;
    Ok(mask)
}

/// Spark's `union` (UNION ALL) of two frames by position: the chunks of `top`, then those of `bottom`, column by column, with the
/// names of `top`.  The column types must be equal.  Not in the reference.
pub fn concat_device(top: &DeviceColumns, bottom: &DeviceColumns) -> Result<DeviceColumns, String> {
    if top.cols.len() != bottom.cols.len() {
        return Err("Union can only be performed on tables with compatible column types".to_string());
    }
    let mut out = DeviceColumns { names: top.names.clone(), cols: Vec::with_capacity(top.cols.len()) };
    for (a, b) in top.cols.iter().zip(&bottom.cols) {
        let pair = [*a as *const BdfCol, *b as *const BdfCol];
        let mut c: *mut BdfCol = std::ptr::null_mut();
        check(unsafe { bdf_concat_dev(dev(), 2, pair.as_ptr(), &mut c) })?;
        out.cols.push(c);
    }
    Ok(out)
}

/// Window functions over one `WindowSpec` (src/window.rs:8-22, not in lib.rs; `WindowFunctions`, src/functions/window.rs:1-11, empty
/// bodies): `partition` are column indices of `frame`, `order` (column index, descending) pairs, `calls` (output name, call) with
/// `call.column` a column pointer of `frame` or null for a ranking function.  The rows are sorted once for all calls.  Returns the new
/// columns only, one chunk each in the frame's row order, named by `calls`; the caller appends them as `DataFrame::with_column` does
/// (an existing name is replaced), so the frame's own columns are never copied.  Rules and departures: include/b200df.h.
pub fn window_device(frame: &DeviceColumns, partition: &[usize], order: &[(usize, bool)], calls: &[(String, BdfWindowCall)]) -> Result<DeviceColumns, String> {
    let part: Vec<*const BdfCol> = partition.iter().map(|p| frame.cols[*p] as *const BdfCol).collect();
    let ord: Vec<BdfSortKey> = order.iter().map(|(c, d)| BdfSortKey { column: frame.cols[*c], descending: *d as i32 }).collect();
    let spec: Vec<BdfWindowCall> = calls.iter().map(|(_, c)| *c).collect();
    let mut out = vec![std::ptr::null_mut(); spec.len()];
    check(unsafe { bdf_window_dev(dev(), part.len() as i32, part.as_ptr(), ord.len() as i32, ord.as_ptr(), spec.len() as i32, spec.as_ptr(),
                                  out.as_mut_ptr()) })?;
    Ok(DeviceColumns { names: calls.iter().map(|(n, _)| n.clone()).collect(), cols: out })
}

/// `WindowSpec::rows_between(start, end)` for one aggregate or value function over `column` (Spark's offsets: negative = PRECEDING,
/// 0 = CURRENT ROW, positive = FOLLOWING, `None` = UNBOUNDED), as a call for `window_device`; e.g. a moving average
/// `rows_between(BDF_WIN_AVG, x, Some(-99), Some(0))` or a forward fill with `ignore_nulls = 1` on `BDF_WIN_LAST_VALUE, None, Some(0)`.
pub fn rows_between(function: i32, column: *const BdfCol, start: Option<i64>, end: Option<i64>) -> BdfWindowCall {
    BdfWindowCall { function, frame: BDF_FRAME_ROWS_BETWEEN, column, offset: if function == BDF_WIN_NTH_VALUE { 1 } else { 0 }, default_bits: 0,
                    has_default: 0, ignore_nulls: 0, start: start.unwrap_or(i64::MIN), end: end.unwrap_or(i64::MAX), start_f: 0.0, end_f: 0.0 }
}

/// `WindowSpec::range_between(start, end)` over the single order key: integer / temporal keys take `start` / `end` in the key's unit,
/// Float32 / Float64 keys `start_f` / `end_f` (set them on the returned call; `None` = UNBOUNDED).
pub fn range_between(function: i32, column: *const BdfCol, start: Option<i64>, end: Option<i64>) -> BdfWindowCall {
    BdfWindowCall { frame: BDF_FRAME_RANGE_BETWEEN, start_f: f64::NEG_INFINITY, end_f: f64::INFINITY, ..rows_between(function, column, start, end) }
}

/// `DataFrame::from_csv(path, None)` on the device: a header, ',', the schema inferred from every record, 1024 rows per
/// RecordBatch (`schema`: one dtype per column instead, BDF_UTF8 for a string column).  Utf8 columns are not on the device path and
/// are left out; a caller that needs them reads just those with arrow's CPU reader and a projection
/// (`csv::Reader::new(file, schema, true, None, 1024, Some(utf8_columns))`).
pub fn from_csv_device(path: &str, schema: Option<&[i32]>) -> Result<DeviceColumns, String> {
    let c_path = std::ffi::CString::new(path).map_err(|e| e.to_string())?;
    let opts = BdfCsvOptions { has_header: 1, delimiter: b',', max_records: -1, batch_size: 1024 };
    let (n_schema, dtypes) = schema.map_or((0, std::ptr::null()), |s| (s.len() as i32, s.as_ptr()));
    let mut file: *mut BdfCsv = std::ptr::null_mut();
    check(unsafe { bdf_csv_open(dev(), c_path.as_ptr(), &opts, n_schema, dtypes, &mut file) })?;
    let (mut n_cols, mut n_batches, mut n_rows) = (0i32, 0i64, 0i64);
    let res = (|| {
        check(unsafe { bdf_csv_describe(file, &mut n_cols, &mut n_batches, &mut n_rows) })?;
        let (mut names, mut idx) = (vec![], vec![]);
        for i in 0..n_cols {
            let (mut name, mut dtype, mut nullable) = (std::ptr::null(), 0i32, 0i32);
            check(unsafe { bdf_csv_column(file, i, &mut name, &mut dtype, &mut nullable) })?;
            if dtype >= 0 {
                names.push(unsafe { std::ffi::CStr::from_ptr(name) }.to_string_lossy().into_owned());
                idx.push(i);
            }
        }
        let mut cols = vec![std::ptr::null_mut(); idx.len()];
        check(unsafe { bdf_csv_read(dev(), file, idx.len() as i32, idx.as_ptr(), cols.as_mut_ptr()) })?;
        Ok(DeviceColumns { names, cols })
    })();
    unsafe { bdf_csv_close(dev(), file) };
    res
}

/// `DataFrame::to_csv(path)` / `Evaluate::write(Csv(path, options))` on the device: every column of the frame is formatted on the GPU
/// (floats in their shortest round-trip digits, as Display prints them) and streamed to the file.  `options`: `CsvWriteOptions
/// { has_headers, delimiter }`, which the reference carries but ignores; None is a header and ','.
pub fn to_csv_device(frame: &DeviceColumns, path: &str, options: Option<(bool, u8)>) -> Result<(), String> {
    let c_path = CString::new(path).map_err(|e| e.to_string())?;
    let names: Vec<CString> = frame.names.iter().map(|n| CString::new(n.as_str())).collect::<Result<_, _>>().map_err(|e| e.to_string())?;
    let name_ptrs: Vec<*const c_char> = names.iter().map(|n| n.as_ptr()).collect();
    let cols: Vec<*const BdfCol> = frame.cols.iter().map(|c| *c as *const BdfCol).collect();
    let opts = options.map(|(h, d)| BdfCsvWriteOptions { has_header: h as i32, delimiter: d });
    let p = opts.as_ref().map_or(std::ptr::null(), |o| o as *const BdfCsvWriteOptions);
    check(unsafe { bdf_csv_write(dev(), c_path.as_ptr(), cols.len() as i32, name_ptrs.as_ptr(), cols.as_ptr(), p) })
}

/// `DataFrame::to_json(path)` on the device, as line-delimited JSON: every column is formatted on the GPU (floats in their shortest
/// round-trip digits, ryu's layout) and streamed to the file.  `types`: one per column (kind 0 for a plain column) or None; `lists`:
/// one per column, non-null where the column is a List<T> (its entry in `frame.cols` is then ignored), or None; `explicit_nulls`
/// writes `"name":null` for a NULL member instead of leaving it out.
pub fn to_json_device(frame: &DeviceColumns, path: &str, types: Option<&[BdfTemporalType]>, lists: Option<&[*const BdfList]>,
                      explicit_nulls: bool) -> Result<(), String> {
    let c_path = CString::new(path).map_err(|e| e.to_string())?;
    let names: Vec<CString> = frame.names.iter().map(|n| CString::new(n.as_str())).collect::<Result<_, _>>().map_err(|e| e.to_string())?;
    let name_ptrs: Vec<*const c_char> = names.iter().map(|n| n.as_ptr()).collect();
    let cols: Vec<*const BdfCol> = frame.cols.iter().enumerate()
        .map(|(j, c)| if lists.map_or(false, |l| !l[j].is_null()) { std::ptr::null() } else { *c as *const BdfCol }).collect();
    let opts = BdfJsonWriteOptions { explicit_nulls: explicit_nulls as i32 };
    check(unsafe {
        bdf_json_write(dev(), c_path.as_ptr(), cols.len() as i32, name_ptrs.as_ptr(), cols.as_ptr(), types.map_or(std::ptr::null(), |t| t.as_ptr()),
                       lists.map_or(std::ptr::null(), |l| l.as_ptr()), &opts)
    })
}

/// DataFrame::to_parquet on the device: every column's pages encoded (and snappy-compressed) on the GPU and streamed to the file.
/// `types`: one per column (kind 0 for a plain column) or None; `options`: None for the defaults.
pub fn to_parquet_device(frame: &DeviceColumns, path: &str, types: Option<&[BdfTemporalType]>,
                         options: Option<BdfParquetWriteOptions>) -> Result<(), String> {
    let c_path = CString::new(path).map_err(|e| e.to_string())?;
    let names: Vec<CString> = frame.names.iter().map(|n| CString::new(n.as_str())).collect::<Result<_, _>>().map_err(|e| e.to_string())?;
    let name_ptrs: Vec<*const c_char> = names.iter().map(|n| n.as_ptr()).collect();
    let cols: Vec<*const BdfCol> = frame.cols.iter().map(|c| *c as *const BdfCol).collect();
    if let Some(t) = types {
        if t.len() != cols.len() { return Err("one temporal type per column".to_string()); }
    }
    let t = types.map_or(std::ptr::null(), |t| t.as_ptr());
    let p = options.as_ref().map_or(std::ptr::null(), |o| o as *const BdfParquetWriteOptions);
    check(unsafe { bdf_parquet_write(dev(), c_path.as_ptr(), cols.len() as i32, name_ptrs.as_ptr(), cols.as_ptr(), t, p) })
}

/// `Column::hist(nbins, density)` on the device (include/b200df.h "distributions"): numpy.histogram's equal-width bins over the
/// valid non-NaN values; `range` None is their [min, max].  Returns (edges, counts or numpy's density).
pub fn hist_device(frame: &DeviceColumns, col: usize, nbins: i32, density: bool, range: Option<(f64, f64)>) -> Result<(Vec<f64>, Vec<f64>), String> {
    let n = nbins.max(0) as usize;
    let (mut edges, mut counts) = (vec![0f64; n + 1], vec![0i64; n]);
    let r = range.map(|(lo, hi)| [lo, hi]);
    let rp = r.as_ref().map_or(std::ptr::null(), |r| r.as_ptr());
    check(unsafe { bdf_hist_dev(dev(), frame.cols[col], nbins, rp, edges.as_mut_ptr(), counts.as_mut_ptr()) })?;
    if !density { return Ok((edges, counts.iter().map(|c| *c as f64).collect())); }
    let mut d = vec![0f64; n];
    check(unsafe { bdf_hist_density(nbins, edges.as_ptr(), counts.as_ptr(), d.as_mut_ptr()) })?;
    Ok((edges, d))
}

/// `Column::uniques()` on the device: the distinct valid values in ascending order as a one-chunk column (and their row counts).
pub fn uniques_device(frame: &DeviceColumns, col: usize, with_counts: bool) -> Result<(*mut BdfCol, Option<*mut BdfCol>), String> {
    let (mut values, mut counts): (*mut BdfCol, *mut BdfCol) = (std::ptr::null_mut(), std::ptr::null_mut());
    let cp = if with_counts { &mut counts as *mut *mut BdfCol } else { std::ptr::null_mut() };
    check(unsafe { bdf_uniques_dev(dev(), frame.cols[col], &mut values, cp) })?;
    Ok((values, if with_counts { Some(counts) } else { None }))
}

/// A run of Float64 Calculations whose intermediates are not kept (config 2: h = sin(((a+b)*c)/d)) as one pass.
/// `inputs` are column indices; node k writes slot inputs.len() + k (see include/b200df.h, bdf_eval_expr_dev).
pub fn fused_chain(frame: &DeviceColumns, inputs: &[usize], nodes: &[BdfExprNode]) -> Result<*mut BdfCol, String> {
    let cols: Vec<*const BdfCol> = inputs.iter().map(|i| frame.cols[*i] as *const BdfCol).collect();
    let mut out: *mut BdfCol = std::ptr::null_mut();
    check(unsafe { bdf_eval_expr_dev(dev(), cols.len() as i32, cols.as_ptr(), nodes.len() as i32, nodes.as_ptr(), &mut out) })?;
    Ok(out)
}

fn check(st: i32) -> Result<(), String> {
    if st == BDF_OK { Ok(()) } else { Err(last_error()) }
}
