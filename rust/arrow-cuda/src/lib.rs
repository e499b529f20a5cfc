//! `arrow-cuda`: drop-in for the `arrow::compute` hot path, backed by hand-written sm_90a kernels
//! (libarrow_cuda.so, C ABI in include/arrow_cuda.h).
//!
//! SOURCE ONLY in this repository — there is no Rust toolchain in the build image, so this crate is written to be correct by
//! inspection; the compiled, GPU-tested equivalents of this layer are `arrow-rs_b200/host/arrow_cuda.hpp` (C++) and
//! `arrow-rs_b200/acu` (Python). A caller switches by changing `use arrow::compute::...` to `use arrow_cuda::compute::...`:
//! every public function below has the reference's name, argument types and result type
//! (arrow/src/compute/mod.rs:20-40, arrow/src/compute/kernels.rs:20-34):
//!
//!   compute::{filter, filter_record_batch, FilterBuilder, FilterPredicate}   arrow-select/src/filter.rs:201-533
//!   compute::{take, take_arrays, take_record_batch, TakeOptions}             arrow-select/src/take.rs:89-164,1123
//!   compute::kernels::numeric::{add .. rem, neg, neg_wrapping}               arrow-arith/src/numeric.rs:36-186
//!   compute::kernels::cmp::{eq .. not_distinct}                              arrow-ord/src/cmp.rs:79-202
//!   compute::kernels::boolean::{and .. is_not_null}                          arrow-arith/src/boolean.rs:60-354
//!   compute::{cast, cast_with_options, CastOptions}                          arrow-cast/src/cast/mod.rs:347,790
//!   compute::kernels::bitwise::{bitwise_and .. bitwise_not}                  arrow-arith/src/bitwise.rs:25-207
//!   compute::{sum, min, max, sum_checked}                                    arrow-arith/src/aggregate.rs:897-1027
//!   compute::{product, product_checked, bit_and, bit_or, bit_xor}            arrow-arith/src/aggregate.rs:788-1001
//!   compute::aggregate::{min_string .. max_fixed_size_binary, min_boolean,   arrow-arith/src/aggregate.rs:372-568, 880-889
//!                        max_boolean, bool_and, bool_or}
//!   compute::{nullif, zip, concat, concat_batches}                           arrow-select/src/{nullif,zip,concat}.rs
//!
//! The wrappers are reference-shaped: host `ArrayRef` in, host `ArrayRef` out, upload / download around every call. A
//! production integration keeps columns in [`DeviceBuffer`]s between calls (what the C++ mirror does); the device-resident
//! building blocks are public for that purpose ([`DeviceArray`], [`Context`]).
pub mod error;
pub mod ffi;

use arrow_array::{make_array, Array, ArrayRef, ArrowPrimitiveType, BooleanArray, Datum, PrimitiveArray, RecordBatch};
use arrow_buffer::{BooleanBuffer, Buffer, MutableBuffer, NullBuffer};
use arrow_data::ArrayData;
use arrow_schema::{ArrowError, DataType, SchemaRef};
use std::cell::RefCell;
use std::os::raw::c_void;
use std::rc::Rc;
use std::sync::Arc;

// ---------------------------------------------------------------------------------------------------------------------
// Context + DeviceBuffer
// ---------------------------------------------------------------------------------------------------------------------
struct ContextInner { raw: *mut ffi::acu_ctx }
impl Drop for ContextInner { fn drop(&mut self) { unsafe { ffi::acu_ctx_destroy(self.raw) } } }

/// One device + one stream (`acu_ctx`). The reference kernels are pure functions; the context is the implicit "where does
/// this run". `Rc`: a ctx must not be used from two threads at once (include/arrow_cuda.h), so it is neither Send nor Sync;
/// every thread gets its own default context.
#[derive(Clone)]
pub struct Context { inner: Rc<ContextInner> }

thread_local! { static DEFAULT: RefCell<Option<Context>> = RefCell::new(None); }

impl Context {
    pub fn new(device: i32) -> Result<Self, ArrowError> {
        let mut raw = std::ptr::null_mut();
        match unsafe { ffi::acu_ctx_create(device, &mut raw) } {
            ffi::ACU_OK => Ok(Self { inner: Rc::new(ContextInner { raw }) }),
            st => Err(ArrowError::ExternalError(format!("acu_ctx_create failed ({st}): no CUDA device, and there is no CPU fallback").into())),
        }
    }
    /// The calling thread's default context (device `ARROW_CUDA_DEVICE`, default 0), created on first use — what the
    /// reference-shaped free functions run on.
    pub fn current() -> Result<Self, ArrowError> {
        DEFAULT.with(|d| {
            if d.borrow().is_none() {
                let dev = std::env::var("ARROW_CUDA_DEVICE").ok().and_then(|s| s.parse().ok()).unwrap_or(0);
                *d.borrow_mut() = Some(Context::new(dev)?);
            }
            Ok(d.borrow().as_ref().unwrap().clone())
        })
    }
    pub(crate) fn raw(&self) -> *mut ffi::acu_ctx { self.inner.raw }
    pub(crate) fn check(&self, st: ffi::acu_status) -> Result<(), ArrowError> {
        if st == ffi::ACU_OK { return Ok(()); }
        Err(error::from_detail(st, unsafe { &*ffi::acu_last_error(self.inner.raw) }))
    }
}

/// DeviceBuffer: `arrow_buffer::Buffer { data: Arc<Bytes>, ptr, length }` (arrow-buffer/src/buffer/immutable.rs:83-96) with
/// the bytes in HBM. It keeps its context alive (the `Rc<ContextInner>`), so it can never be freed on a destroyed ctx.
pub struct DeviceBuffer { ctx: Context, ptr: *mut c_void, len: usize }
impl DeviceBuffer {
    /// `len` bytes (+ 16 bytes of slack: kernels read whole aligned words), uninitialised.
    pub fn allocate(ctx: &Context, len: usize) -> Result<Self, ArrowError> {
        let mut ptr = std::ptr::null_mut();
        ctx.check(unsafe { ffi::acu_malloc(ctx.raw(), len + 16, &mut ptr) })?;
        Ok(Self { ctx: ctx.clone(), ptr, len })
    }
    pub fn from_host(ctx: &Context, bytes: &[u8]) -> Result<Self, ArrowError> {
        let b = Self::allocate(ctx, bytes.len())?;
        if !bytes.is_empty() {
            ctx.check(unsafe { ffi::acu_memcpy_h2d(ctx.raw(), b.ptr, bytes.as_ptr() as *const c_void, bytes.len()) })?;
        }
        Ok(b)
    }
    /// The first `len` bytes as an arrow `Buffer` (128-byte aligned `MutableBuffer`, so any native type can view it).
    pub fn to_host(&self, len: usize) -> Result<Buffer, ArrowError> {
        let len = len.min(self.len);
        let mut m = MutableBuffer::from_len_zeroed(len);
        if len > 0 {
            self.ctx.check(unsafe { ffi::acu_memcpy_d2h(self.ctx.raw(), m.as_mut_ptr() as *mut c_void, self.ptr, len) })?;
        }
        Ok(m.into())
    }
    pub fn as_ptr(&self) -> *mut c_void { self.ptr }
    pub fn len(&self) -> usize { self.len }
    pub fn is_empty(&self) -> bool { self.len == 0 }
}
impl Drop for DeviceBuffer { fn drop(&mut self) { unsafe { ffi::acu_free(self.ctx.raw(), self.ptr); } } }

fn bitmap_bytes(rows: usize) -> usize { (rows + 63) / 64 * 8 }

// ---------------------------------------------------------------------------------------------------------------------
// Host array -> device view (generic over the array kinds of the hot path, via ArrayData's buffer layout)
// ---------------------------------------------------------------------------------------------------------------------
/// acu_dtype code of a numeric DataType (the order of include/arrow_cuda.h `acu_dtype`).
fn dtype_code(t: &DataType) -> Option<i32> {
    Some(match t {
        DataType::Int8 => ffi::ACU_I8, DataType::Int16 => ffi::ACU_I16, DataType::Int32 => ffi::ACU_I32, DataType::Int64 => ffi::ACU_I64,
        DataType::UInt8 => ffi::ACU_U8, DataType::UInt16 => ffi::ACU_U16, DataType::UInt32 => ffi::ACU_U32, DataType::UInt64 => ffi::ACU_U64,
        DataType::Float32 => ffi::ACU_F32, DataType::Float64 => ffi::ACU_F64,
        _ => return None,
    })
}

/// acu_dtype of a type's native for acu_cmp / acu_neg / the aggregates: the numeric types, and decimals as their integers
/// (the reference compares and aggregates decimals as their natives). acu_arith takes only `dtype_code`.
fn native_code(t: &DataType) -> Option<i32> {
    match t {
        DataType::Decimal32(_, _) => Some(ffi::ACU_I32),
        DataType::Decimal64(_, _) => Some(ffi::ACU_I64),
        DataType::Decimal128(_, _) => Some(ffi::ACU_I128),
        t => dtype_code(t),
    }
}

/// acu_decimal_type of Decimal32 / 64 / 128 (Decimal256 is not supported on the device)
fn decimal_type(t: &DataType) -> Option<ffi::acu_decimal_type> {
    let (byte_width, precision, scale) = match t {
        DataType::Decimal32(p, s) => (4, *p, *s),
        DataType::Decimal64(p, s) => (8, *p, *s),
        DataType::Decimal128(p, s) => (16, *p, *s),
        _ => return None,
    };
    Some(ffi::acu_decimal_type { byte_width, precision, scale, reserved: [0; 2] })
}

enum Kind { Primitive(usize), Boolean, Bytes(usize), FixedSizeBinary(usize) }
fn kind_of(t: &DataType) -> Result<Kind, ArrowError> {
    match t {
        DataType::Boolean => Ok(Kind::Boolean),
        DataType::Utf8 | DataType::Binary => Ok(Kind::Bytes(4)),
        DataType::LargeUtf8 | DataType::LargeBinary => Ok(Kind::Bytes(8)),
        DataType::FixedSizeBinary(w) if *w >= 0 => Ok(Kind::FixedSizeBinary(*w as usize)),
        // filter / take are type-agnostic copies: every fixed-width primitive goes by element width (SURVEY.md §8(a))
        t => t.primitive_width().map(Kind::Primitive).ok_or_else(|| ArrowError::NotYetImplemented(format!("arrow-cuda: data type {t}"))),
    }
}

/// A host array uploaded to HBM: owns the device copies, `column` is the borrowed view the C ABI takes.
pub struct DeviceArray {
    _bufs: Vec<DeviceBuffer>,
    pub column: ffi::acu_column,
    data_bytes: usize,
}

impl DeviceArray {
    pub fn upload(ctx: &Context, array: &dyn Array, is_scalar: bool) -> Result<Self, ArrowError> {
        let d: ArrayData = array.to_data();
        let kind = kind_of(d.data_type())?;
        let mut bufs = Vec::new();
        let (validity, validity_offset, null_count) = match d.nulls() {
            Some(n) => {
                let b = DeviceBuffer::from_host(ctx, n.buffer().as_slice())?;
                let p = b.as_ptr() as *const u8;
                bufs.push(b);
                (p, n.offset() as i64, n.null_count() as i64)
            }
            None => (std::ptr::null(), 0, 0),
        };
        let mut a = ffi::acu_array { values: std::ptr::null(), values_offset: 0, validity, validity_offset, len: d.len() as i64,
                                     null_count, is_scalar: is_scalar as i32, reserved: 0 };
        let mut col = ffi::acu_column { kind: ffi::ACU_COL_PRIMITIVE, width: 0, array: a, data: std::ptr::null() };
        let mut data_bytes = 0;
        match kind {
            Kind::Primitive(w) => {
                let bytes = &d.buffers()[0].as_slice()[d.offset() * w..(d.offset() + d.len()) * w];
                let b = DeviceBuffer::from_host(ctx, bytes)?;
                a.values = b.as_ptr();
                bufs.push(b);
                col.width = w as i32;
            }
            Kind::Boolean => {
                let b = DeviceBuffer::from_host(ctx, d.buffers()[0].as_slice())?;
                a.values = b.as_ptr();
                a.values_offset = d.offset() as i64;
                bufs.push(b);
                col.kind = ffi::ACU_COL_BOOLEAN;
            }
            Kind::Bytes(ob) => {
                let offs = &d.buffers()[0].as_slice()[d.offset() * ob..(d.offset() + d.len() + 1) * ob];
                let o = DeviceBuffer::from_host(ctx, offs)?;
                let v = DeviceBuffer::from_host(ctx, d.buffers()[1].as_slice())?;
                a.values = o.as_ptr();
                col.data = v.as_ptr() as *const u8;
                data_bytes = v.len();
                bufs.push(o);
                bufs.push(v);
                col.kind = ffi::ACU_COL_BYTES;
                col.width = ob as i32;
            }
            Kind::FixedSizeBinary(w) => {  // values from logical row 0 (any alignment)
                let bytes = &d.buffers()[0].as_slice()[d.offset() * w..(d.offset() + d.len()) * w];
                let b = DeviceBuffer::from_host(ctx, bytes)?;
                a.values = b.as_ptr();
                bufs.push(b);
                col.kind = ffi::ACU_COL_FIXED_SIZE_BINARY;
                col.width = w as i32;
            }
        }
        col.array = a;
        Ok(Self { _bufs: bufs, column: col, data_bytes })
    }
    fn view(&self) -> &ffi::acu_array { &self.column.array }
}

/// Caller-owned output of one column + the download back into an `ArrayRef` of `data_type`.
struct ColumnOut { values: DeviceBuffer, validity: DeviceBuffer, data: Option<DeviceBuffer>, out: ffi::acu_column_out }
impl ColumnOut {
    fn new(ctx: &Context, data_type: &DataType, rows: usize, data_capacity: usize) -> Result<Self, ArrowError> {
        let vbytes = match kind_of(data_type)? {
            Kind::Primitive(w) => rows.max(1) * w,
            Kind::Boolean => bitmap_bytes(rows.max(1)),
            Kind::Bytes(ob) => (rows + 1) * ob,
            Kind::FixedSizeBinary(w) => (rows * w).max(1),
        };
        let values = DeviceBuffer::allocate(ctx, vbytes)?;
        let validity = DeviceBuffer::allocate(ctx, bitmap_bytes(rows.max(1)))?;
        let data = match kind_of(data_type)? { Kind::Bytes(_) => Some(DeviceBuffer::allocate(ctx, data_capacity)?), _ => None };
        let out = ffi::acu_column_out {
            array: ffi::acu_array_out { values: values.as_ptr(), validity: validity.as_ptr() as *mut u8, len: 0, null_count: 0, has_validity: 0, reserved: 0 },
            data: data.as_ref().map_or(std::ptr::null_mut(), |d| d.as_ptr() as *mut u8),
            data_capacity: data_capacity as i64,
            data_len: 0,
        };
        Ok(Self { values, validity, data, out })
    }
    fn array_out(&mut self) -> *mut ffi::acu_array_out { &mut self.out.array }
    fn finish(&self, data_type: &DataType) -> Result<ArrayRef, ArrowError> {
        let o = &self.out.array;
        let len = o.len as usize;
        let nulls = if o.has_validity != 0 {
            let bits = BooleanBuffer::new(self.validity.to_host(bitmap_bytes(len))?, 0, len);
            Some(unsafe { NullBuffer::new_unchecked(bits, o.null_count as usize) })
        } else { None };
        let mut b = ArrayData::builder(data_type.clone()).len(len).nulls(nulls);
        match kind_of(data_type)? {
            Kind::Primitive(w) => { b = b.add_buffer(self.values.to_host(len * w)?); }
            Kind::Boolean => { b = b.add_buffer(self.values.to_host(bitmap_bytes(len))?); }
            Kind::FixedSizeBinary(w) => { b = b.add_buffer(self.values.to_host(len * w)?); }
            Kind::Bytes(ob) => {
                b = b.add_buffer(self.values.to_host((len + 1) * ob)?);
                b = b.add_buffer(self.data.as_ref().unwrap().to_host(self.out.data_len as usize)?);
            }
        }
        // the kernels produce valid Arrow buffers (bit-exact with the reference, tests/): no second validation pass
        Ok(make_array(unsafe { b.build_unchecked() }))
    }
}

fn numeric_dtype(ctx_what: &str, t: &DataType) -> Result<i32, ArrowError> {
    dtype_code(t).ok_or_else(|| ArrowError::InvalidArgumentError(format!("Invalid {ctx_what} operation: {t}")))
}

// ---------------------------------------------------------------------------------------------------------------------
// compute — the reference's public names and signatures
// ---------------------------------------------------------------------------------------------------------------------
pub mod compute {
    use super::*;

    // ---- filter (arrow-select/src/filter.rs) ------------------------------------------------------------------------
    /// RAII owner of the device-resident plan (`FilterPredicate`, filter.rs:442-533): freed on every path.
    struct Plan { ctx: Context, raw: *mut ffi::acu_filter_plan }
    impl Drop for Plan { fn drop(&mut self) { unsafe { ffi::acu_filter_plan_destroy(self.ctx.raw(), self.raw) } } }

    /// `FilterBuilder` (filter.rs:254-324). `optimize()` is a no-op here: the plan is always the "optimized" form.
    pub struct FilterBuilder { predicate: BooleanArray }
    impl FilterBuilder {
        pub fn new(filter: &BooleanArray) -> Self { Self { predicate: filter.clone() } }
        pub fn optimize(self) -> Self { self }
        pub fn build(self) -> Result<FilterPredicate, ArrowError> {
            let ctx = Context::current()?;
            let p = DeviceArray::upload(&ctx, &self.predicate, false)?;
            let mut raw = std::ptr::null_mut();
            ctx.check(unsafe { ffi::acu_filter_plan_create(ctx.raw(), p.view(), &mut raw) })?;
            Ok(FilterPredicate { plan: Plan { ctx, raw } })
        }
    }

    /// `FilterPredicate` (filter.rs:442-533): one scan of the predicate, reused for any number of arrays / batches.
    pub struct FilterPredicate { plan: Plan }
    impl FilterPredicate {
        /// Number of rows selected (FilterPredicate::count).
        pub fn count(&self) -> usize { unsafe { ffi::acu_filter_plan_count(self.plan.raw) as usize } }
        pub fn filter(&self, values: &dyn Array) -> Result<ArrayRef, ArrowError> {
            let ctx = &self.plan.ctx;
            if let DataType::List(_) | DataType::LargeList(_) | DataType::FixedSizeList(_, _) = values.data_type() {
                return list::filter(ctx, self.plan.raw, values, None);
            }
            if let DataType::RunEndEncoded(_, _) = values.data_type() {
                return run_end::filter(ctx, self.plan.raw, values);
            }
            if let DataType::Struct(_) | DataType::Union(_, _) = values.data_type() {
                return nested::filter(ctx, self.plan.raw, values, None);
            }
            let v = DeviceArray::upload(ctx, values, false)?;
            let mut out = ColumnOut::new(ctx, values.data_type(), self.count(), v.data_bytes)?;
            let st = match kind_of(values.data_type())? {
                Kind::Primitive(w) => unsafe { ffi::acu_filter_primitive(ctx.raw(), self.plan.raw, w as i32, v.view(), out.array_out()) },
                Kind::Boolean => unsafe { ffi::acu_filter_boolean(ctx.raw(), self.plan.raw, v.view(), out.array_out()) },
                // filter_fixed_size_binary (filter.rs:946-996)
                Kind::FixedSizeBinary(w) => unsafe {
                    ffi::acu_filter_fixed_size_binary(ctx.raw(), self.plan.raw, w as i32, v.view(), out.array_out())
                },
                Kind::Bytes(ob) => unsafe {
                    ffi::acu_filter_bytes(ctx.raw(), self.plan.raw, ob as i32, v.view().values, v.column.data, v.view(), out.out.array.values,
                                          out.out.data, out.out.data_capacity, &mut out.out.data_len, &mut out.out.array)
                },
            };
            ctx.check(st)?;
            out.finish(values.data_type())
        }
        /// filter.rs:459-478: every column with the same plan, one stream synchronisation per 64 columns.
        pub fn filter_record_batch(&self, record_batch: &RecordBatch) -> Result<RecordBatch, ArrowError> {
            let ctx = &self.plan.ctx;
            let n = record_batch.num_columns();
            let ups = record_batch.columns().iter().map(|c| DeviceArray::upload(ctx, c.as_ref(), false)).collect::<Result<Vec<_>, _>>()?;
            let mut outs = record_batch.columns().iter().zip(&ups).map(|(c, u)| ColumnOut::new(ctx, c.data_type(), self.count(), u.data_bytes))
                .collect::<Result<Vec<_>, _>>()?;
            for first in (0..n).step_by(ffi::ACU_MAX_BATCH_COLUMNS) {
                let last = (first + ffi::ACU_MAX_BATCH_COLUMNS).min(n);
                let cols: Vec<ffi::acu_column> = ups[first..last].iter().map(|u| u.column).collect();
                let mut raw: Vec<ffi::acu_column_out> = outs[first..last].iter().map(|o| o.out).collect();
                ctx.check(unsafe { ffi::acu_filter_record_batch(ctx.raw(), self.plan.raw, (last - first) as i32, cols.as_ptr(), raw.as_mut_ptr()) })?;
                for (o, r) in outs[first..last].iter_mut().zip(raw) { o.out = r; }
            }
            let cols = record_batch.columns().iter().zip(&outs).map(|(c, o)| o.finish(c.data_type())).collect::<Result<Vec<_>, _>>()?;
            RecordBatch::try_new(record_batch.schema(), cols)
        }
    }

    /// `arrow::compute::filter` (filter.rs:201-213).
    pub fn filter(values: &dyn Array, predicate: &BooleanArray) -> Result<ArrayRef, ArrowError> {
        FilterBuilder::new(predicate).build()?.filter(values)
    }
    /// `arrow::compute::filter_record_batch` (filter.rs:225-244).
    pub fn filter_record_batch(record_batch: &RecordBatch, predicate: &BooleanArray) -> Result<RecordBatch, ArrowError> {
        FilterBuilder::new(predicate).build()?.filter_record_batch(record_batch)
    }

    // ---- take (arrow-select/src/take.rs) ------------------------------------------------------------------------------
    /// take.rs:388-394
    #[derive(Clone, Debug, Default)]
    pub struct TakeOptions { pub check_bounds: bool }

    fn index_dtype(indices: &dyn Array) -> Result<i32, ArrowError> {
        match indices.data_type() {  // take.rs:96-104 downcast_integer_array!
            DataType::Float32 | DataType::Float64 => None,
            t => dtype_code(t),
        }.ok_or_else(|| ArrowError::InvalidArgumentError(format!("Take only supported for integers, got {:?}", indices.data_type())))
    }

    /// `arrow::compute::take` (take.rs:89-105).
    pub fn take(values: &dyn Array, indices: &dyn Array, options: Option<TakeOptions>) -> Result<ArrayRef, ArrowError> {
        let ctx = Context::current()?;
        let idt = index_dtype(indices)?;
        let check = options.unwrap_or_default().check_bounds as i32;
        if let DataType::List(_) | DataType::LargeList(_) | DataType::FixedSizeList(_, _) = values.data_type() {
            return list::take(&ctx, values, indices, idt, check, false);
        }
        if let DataType::RunEndEncoded(_, _) = values.data_type() {
            return run_end::take(&ctx, values, indices, idt, check);
        }
        if let DataType::Struct(_) | DataType::Union(_, _) = values.data_type() {
            return nested::take(&ctx, values, indices, idt, check, false);
        }
        let (v, ix) = (DeviceArray::upload(&ctx, values, false)?, DeviceArray::upload(&ctx, indices, false)?);
        let m = indices.len();
        let st;
        let mut out;
        match kind_of(values.data_type())? {
            Kind::Primitive(w) => {
                out = ColumnOut::new(&ctx, values.data_type(), m, 0)?;
                st = unsafe { ffi::acu_take_primitive(ctx.raw(), w as i32, v.view(), ix.view(), idt, check, out.array_out()) };
            }
            Kind::Boolean => {
                out = ColumnOut::new(&ctx, values.data_type(), m, 0)?;
                st = unsafe { ffi::acu_take_boolean(ctx.raw(), v.view(), ix.view(), idt, check, out.array_out()) };
            }
            Kind::FixedSizeBinary(w) => {  // take_fixed_size_binary (take.rs:802-862)
                out = ColumnOut::new(&ctx, values.data_type(), m, 0)?;
                st = unsafe { ffi::acu_take_fixed_size_binary(ctx.raw(), w as i32, v.view(), ix.view(), idt, check, out.array_out()) };
            }
            Kind::Bytes(ob) => {
                // two-phase: offsets + required bytes first, then the copy (take_bytes computes the capacity first too, take.rs:520-523)
                let mut probe = ColumnOut::new(&ctx, values.data_type(), m, 0)?;
                let mut need = 0i64;
                ctx.check(unsafe {
                    ffi::acu_take_bytes(ctx.raw(), ob as i32, v.view().values, v.column.data, v.view(), ix.view(), idt, check, probe.out.array.values,
                                        std::ptr::null_mut(), 0, &mut need, &mut probe.out.array)
                })?;
                out = ColumnOut::new(&ctx, values.data_type(), m, need as usize)?;
                st = unsafe {
                    ffi::acu_take_bytes(ctx.raw(), ob as i32, v.view().values, v.column.data, v.view(), ix.view(), idt, check, out.out.array.values,
                                        out.out.data, out.out.data_capacity, &mut out.out.data_len, &mut out.out.array)
                };
            }
        }
        ctx.check(st)?; // ACU_ERR_PANIC_OUT_OF_BOUNDS panics inside, like take.rs:447
        out.finish(values.data_type())
    }
    // ---- RunEndEncoded (filter_run_end_array filter.rs:628-677, take_run take.rs:948-995) -----------------------------
    /// acu_filter_run_end / acu_take_run_end write the new run ends and return the plan / value indices of the values child,
    /// which then goes through filter / take of its own type.
    mod run_end {
        use super::*;
        use arrow_array::cast::AsArray;
        use arrow_array::types::{Int16Type, Int32Type, Int64Type, RunEndIndexType, UInt32Type, UInt64Type};
        use arrow_array::{new_empty_array, Array, RunArray};
        use arrow_buffer::ScalarBuffer;

        struct Ree { r: ffi::acu_run_array, width: usize, _ends: DeviceBuffer }

        fn describe<R: RunEndIndexType>(ctx: &Context, a: &RunArray<R>) -> Result<Ree, ArrowError> {
            let ends = a.run_ends();
            let dev = DeviceBuffer::from_host(ctx, ends.inner().inner().as_slice())?;
            let r = ffi::acu_run_array { run_end_dtype: dtype_code(&R::DATA_TYPE).unwrap(), reserved: 0, run_ends: dev.as_ptr(),
                                         n_runs: ends.values().len() as i64, offset: ends.offset() as i64, len: ends.len() as i64 };
            Ok(Ree { r, width: std::mem::size_of::<R::Native>(), _ends: dev })
        }

        fn run_array<R: RunEndIndexType>(ends: &DeviceBuffer, runs: usize, width: usize, values: &dyn Array) -> Result<ArrayRef, ArrowError> {
            let re = PrimitiveArray::<R>::new(ScalarBuffer::new(ends.to_host(runs * width)?, 0, runs), None);
            Ok(Arc::new(RunArray::<R>::try_new(&re, values)?))
        }

        pub(super) fn filter(ctx: &Context, plan: *mut ffi::acu_filter_plan, values: &dyn Array) -> Result<ArrayRef, ArrowError> {
            match values.data_type() {
                DataType::RunEndEncoded(f, _) => match f.data_type() {
                    DataType::Int16 => filter_typed(ctx, plan, values.as_run::<Int16Type>()),
                    DataType::Int32 => filter_typed(ctx, plan, values.as_run::<Int32Type>()),
                    _ => filter_typed(ctx, plan, values.as_run::<Int64Type>()),
                },
                _ => unreachable!(),
            }
        }

        fn filter_typed<R: RunEndIndexType>(ctx: &Context, plan: *mut ffi::acu_filter_plan, a: &RunArray<R>) -> Result<ArrayRef, ArrowError> {
            let d = describe(ctx, a)?;
            let count = unsafe { ffi::acu_filter_plan_count(plan) } as usize;
            let ends = DeviceBuffer::allocate(ctx, count.min(a.run_ends().values().len()).max(1) * d.width)?;
            let (mut runs, mut start, mut vplan) = (0i64, 0i64, std::ptr::null_mut());
            ctx.check(unsafe { ffi::acu_filter_run_end(ctx.raw(), plan, &d.r, ends.as_ptr(), &mut runs, &mut start, &mut vplan) })?;
            if vplan.is_null() {  // filter.rs:545-546: new_empty_array / values.slice(0, count)
                return Ok(if unsafe { ffi::acu_filter_plan_strategy(plan) } == 1 { Array::slice(a, 0, count) } else { new_empty_array(a.data_type()) });
            }
            let vplan = Plan { ctx: ctx.clone(), raw: vplan };
            let vlen = unsafe { ffi::acu_filter_plan_len(vplan.raw) } as usize;
            let v = FilterPredicate { plan: vplan }.filter(a.values().slice(start as usize, vlen).as_ref())?;
            run_array::<R>(&ends, runs as usize, d.width, v.as_ref())
        }

        pub(super) fn take(ctx: &Context, values: &dyn Array, indices: &dyn Array, idt: i32, check: i32) -> Result<ArrayRef, ArrowError> {
            match values.data_type() {
                DataType::RunEndEncoded(f, _) => match f.data_type() {
                    DataType::Int16 => take_typed(ctx, values.as_run::<Int16Type>(), indices, idt, check),
                    DataType::Int32 => take_typed(ctx, values.as_run::<Int32Type>(), indices, idt, check),
                    _ => take_typed(ctx, values.as_run::<Int64Type>(), indices, idt, check),
                },
                _ => unreachable!(),
            }
        }

        fn take_typed<R: RunEndIndexType>(ctx: &Context, a: &RunArray<R>, indices: &dyn Array, idt: i32, check: i32) -> Result<ArrayRef, ArrowError> {
            let d = describe(ctx, a)?;
            let vals = a.values();
            let mut rv: ffi::acu_run_values = unsafe { std::mem::zeroed() };
            let _up = match vals.data_type() {
                DataType::List(_) | DataType::LargeList(_) | DataType::FixedSizeList(_, _) | DataType::RunEndEncoded(_, _)
                | DataType::Struct(_) | DataType::Union(_, _) | DataType::FixedSizeBinary(_) => {  // (the run merge compares values)
                    rv.kind = ffi::ACU_RUN_VALUES_NESTED;
                    None
                }
                t => {
                    let u = DeviceArray::upload(ctx, vals.as_ref(), false)?;
                    match kind_of(t)? {
                        Kind::Primitive(w) => { rv.kind = ffi::ACU_RUN_VALUES_FIXED; rv.width = w as i32; rv.array = *u.view(); }
                        Kind::Boolean => { rv.kind = ffi::ACU_RUN_VALUES_BOOLEAN; rv.array = *u.view(); }
                        Kind::FixedSizeBinary(_) => unreachable!(),
                        Kind::Bytes(ob) => {
                            rv.kind = ffi::ACU_RUN_VALUES_BYTES;
                            rv.width = ob as i32;
                            rv.bytes = ffi::acu_bytes_array { offsets: u.view().values, data: u.column.data, nulls: *u.view() };
                        }
                    }
                    Some(u)
                }
            };
            let ix = DeviceArray::upload(ctx, indices, false)?;
            let m = indices.len();
            let wide = matches!(indices.data_type(), DataType::Int64 | DataType::UInt64);  // ToIndices: UInt64 value indices
            let ends = DeviceBuffer::allocate(ctx, m.max(1) * d.width)?;
            let vi = DeviceBuffer::allocate(ctx, m.max(1) * if wide { 8 } else { 4 })?;
            let mut runs = 0i64;
            ctx.check(unsafe { ffi::acu_take_run_end(ctx.raw(), &d.r, &rv, ix.view(), idt, check, ends.as_ptr(), vi.as_ptr(), &mut runs) })?;
            if m == 0 { return Ok(new_empty_array(a.data_type())); }  // take.rs:216-218
            let n = runs as usize;
            let vix: ArrayRef = if wide {
                Arc::new(PrimitiveArray::<UInt64Type>::new(vi.to_host(n * 8)?.into(), None))
            } else {
                Arc::new(PrimitiveArray::<UInt32Type>::new(vi.to_host(n * 4)?.into(), None))
            };
            let v = super::take(vals.as_ref(), vix.as_ref(), None)?;
            run_array::<R>(&ends, n, d.width, v.as_ref())
        }
    }

    // ---- List / LargeList / FixedSizeList (filter.rs:535-625, take.rs:646-795) ----------------------------------------
    /// One C call per level: acu_filter_list / acu_take_list return the child's plan / row map, and the child goes through
    /// filter / take of its own type (these functions again for a nested list). A List's child is extended
    /// (MutableArrayData: a Utf8 / Binary child keeps the bytes under its null rows, acu_take_bytes_extend); a
    /// FixedSizeList's child is taken, and its take_bits panic comes after the child's own errors.
    mod list {
        use super::*;
        use arrow_array::types::{UInt32Type, UInt64Type};
        use arrow_array::{Array, FixedSizeListArray, GenericListArray, OffsetSizeTrait};

        struct Level { list: ffi::acu_list_array, child: ArrayRef, ob: usize, _bufs: Vec<DeviceBuffer>, _nulls: DeviceArray }

        fn level(ctx: &Context, values: &dyn Array) -> Result<Level, ArrowError> {
            fn generic<O: OffsetSizeTrait>(ctx: &Context, a: &GenericListArray<O>, kind: i32, bufs: &mut Vec<DeviceBuffer>)
                                           -> Result<(ffi::acu_list_array, ArrayRef, DeviceArray), ArrowError> {
                let offs = DeviceBuffer::from_host(ctx, a.offsets().inner().inner().as_slice())?;
                let nulls = DeviceArray::upload(ctx, &BooleanArray::new(BooleanBuffer::new_set(a.len()), a.nulls().cloned()), false)?;
                let mut l = ffi::acu_list_array { kind, list_size: 0, offsets: offs.as_ptr(), nulls: *nulls.view(), child_len: a.values().len() as i64 };
                l.nulls.values = std::ptr::null();
                bufs.push(offs);
                Ok((l, a.values().clone(), nulls))
            }
            let mut bufs = Vec::new();
            let (list, child, ob, nulls) = match values.data_type() {
                DataType::List(_) => { let (l, c, n) = generic(ctx, values.as_any().downcast_ref::<GenericListArray<i32>>().unwrap(), ffi::ACU_LIST, &mut bufs)?; (l, c, 4, n) }
                DataType::LargeList(_) => { let (l, c, n) = generic(ctx, values.as_any().downcast_ref::<GenericListArray<i64>>().unwrap(), ffi::ACU_LARGE_LIST, &mut bufs)?; (l, c, 8, n) }
                _ => {
                    let a = values.as_any().downcast_ref::<FixedSizeListArray>().unwrap();
                    let nulls = DeviceArray::upload(ctx, &BooleanArray::new(BooleanBuffer::new_set(a.len()), a.nulls().cloned()), false)?;
                    let mut l = ffi::acu_list_array { kind: ffi::ACU_FIXED_SIZE_LIST, list_size: a.value_length(), offsets: std::ptr::null(),
                                                      nulls: *nulls.view(), child_len: a.values().len() as i64 };
                    l.nulls.values = std::ptr::null();
                    (l, a.values().clone(), 0, nulls)
                }
            };
            Ok(Level { list, child, ob, _bufs: bufs, _nulls: nulls })
        }

        fn rebuild(values: &dyn Array, offsets: Option<Buffer>, child: ArrayRef, len: usize, nulls: Option<NullBuffer>) -> ArrayRef {
            let mut b = ArrayData::builder(values.data_type().clone()).len(len).nulls(nulls).add_child_data(child.to_data());
            if let Some(o) = offsets { b = b.add_buffer(o); }
            make_array(unsafe { b.build_unchecked() })
        }

        pub(super) fn nulls_of(validity: &DeviceBuffer, o: &ffi::acu_array_out) -> Result<Option<NullBuffer>, ArrowError> {
            if o.has_validity == 0 { return Ok(None); }
            let bits = BooleanBuffer::new(validity.to_host(bitmap_bytes(o.len as usize))?, 0, o.len as usize);
            Ok(Some(unsafe { NullBuffer::new_unchecked(bits, o.null_count as usize) }))
        }

        /// `child_step`: `values` is a child of a list whose top level was filtered with a plan other than All (None at the
        /// top). The reference builds those levels with MutableArrayData (filter.rs:600), whose freeze drops a NullBuffer
        /// without nulls (arrow-data/src/transform/mod.rs:936) even where the level's own plan selects every row; under a
        /// top-level All it slices every level as it is.
        pub(super) fn filter(ctx: &Context, plan: *mut ffi::acu_filter_plan, values: &dyn Array, child_step: Option<bool>)
                             -> Result<ArrayRef, ArrowError> {
            let lv = level(ctx, values)?;
            let n = unsafe { ffi::acu_filter_plan_count(plan) } as usize;
            let offs = DeviceBuffer::allocate(ctx, (n + 1) * lv.ob.max(1))?;
            let validity = DeviceBuffer::allocate(ctx, bitmap_bytes(n.max(1)))?;
            let mut o = ffi::acu_array_out { values: std::ptr::null_mut(), validity: validity.as_ptr() as *mut u8, len: 0, null_count: 0, has_validity: 0, reserved: 0 };
            let mut child_plan = std::ptr::null_mut();
            ctx.check(unsafe { ffi::acu_filter_list(ctx.raw(), plan, &lv.list, offs.as_ptr(), &mut o, &mut child_plan) })?;
            let child_plan = Plan { ctx: ctx.clone(), raw: child_plan };
            let step = child_step.unwrap_or(n != unsafe { ffi::acu_filter_plan_len(plan) } as usize);
            let child = match lv.child.data_type() {
                DataType::List(_) | DataType::LargeList(_) | DataType::FixedSizeList(_, _) => filter(ctx, child_plan.raw, lv.child.as_ref(), Some(step))?,
                DataType::Struct(_) | DataType::Union(_, _) => nested::filter(ctx, child_plan.raw, lv.child.as_ref(), Some(step))?,
                _ => {
                    let rows = unsafe { ffi::acu_filter_plan_count(child_plan.raw) } as usize;
                    let c = FilterPredicate { plan: child_plan }.filter(lv.child.as_ref())?;
                    if step { keep_width0_rows(drop_empty_nulls(c), rows) } else { c }
                }
            };
            if child_step == Some(true) && o.null_count == 0 { o.has_validity = 0; }
            let offsets = if lv.ob > 0 { Some(offs.to_host((n + 1) * lv.ob)?) } else { None };
            Ok(rebuild(values, offsets, child, n, nulls_of(&validity, &o)?))
        }

        /// MutableArrayData keeps every extended row of a FixedSizeBinary(0) child (try_new's length rule is the top level's)
        fn keep_width0_rows(a: ArrayRef, rows: usize) -> ArrayRef {
            if a.data_type() != &DataType::FixedSizeBinary(0) || a.len() == rows { return a; }
            make_array(unsafe { a.to_data().into_builder().len(rows).build_unchecked() })
        }

        fn drop_empty_nulls(a: ArrayRef) -> ArrayRef {
            if a.nulls().map_or(true, |n| n.null_count() > 0) { return a; }
            make_array(unsafe { a.to_data().into_builder().nulls(None).build_unchecked() })
        }

        pub(super) fn take(ctx: &Context, values: &dyn Array, indices: &dyn Array, idt: i32, check: i32, keep: bool) -> Result<ArrayRef, ArrowError> {
            let lv = level(ctx, values)?;
            let ix = DeviceArray::upload(ctx, indices, false)?;
            let m = indices.len();
            let wide = lv.ob > 0 && lv.list.child_len > u32::MAX as i64;
            let cdt = if wide { 7 } else { 6 }; // ACU_U64 / ACU_U32
            let offs = DeviceBuffer::allocate(ctx, (m + 1) * lv.ob.max(1))?;
            let validity = DeviceBuffer::allocate(ctx, bitmap_bytes(m.max(1)))?;
            let mut o = ffi::acu_array_out { values: std::ptr::null_mut(), validity: validity.as_ptr() as *mut u8, len: 0, null_count: 0, has_validity: 0, reserved: 0 };
            let mut rows = 0i64;
            let mut cn = ffi::acu_array_out { values: std::ptr::null_mut(), validity: std::ptr::null_mut(), len: 0, null_count: 0, has_validity: 0, reserved: 0 };
            ctx.check(unsafe { ffi::acu_take_list(ctx.raw(), &lv.list, ix.view(), idt, check, keep as i32, offs.as_ptr(), &mut o, cdt,
                                                  std::ptr::null_mut(), 0, &mut rows, &mut cn) })?;
            let n = rows as usize;
            let map = DeviceBuffer::allocate(ctx, n.max(1) * if wide { 8 } else { 4 })?;
            let map_valid = DeviceBuffer::allocate(ctx, bitmap_bytes(n.max(1)))?;
            cn.validity = map_valid.as_ptr() as *mut u8;
            let st = unsafe { ffi::acu_take_list(ctx.raw(), &lv.list, ix.view(), idt, check, keep as i32, offs.as_ptr(), &mut o, cdt,
                                                 map.as_ptr(), rows, &mut rows, &mut cn) };
            let deferred = if st != ffi::ACU_OK && lv.ob == 0 { Some(ctx.check(st).unwrap_err()) } else { ctx.check(st).map(|_| None)? };
            let map_nulls = nulls_of(&map_valid, &cn)?;
            let rm: ArrayRef = if wide {
                Arc::new(PrimitiveArray::<UInt64Type>::new(map.to_host(n * 8)?.into(), map_nulls))
            } else {
                Arc::new(PrimitiveArray::<UInt32Type>::new(map.to_host(n * 4)?.into(), map_nulls))
            };
            // a List's child is extended, a FixedSizeList's child is taken
            let child = child_take(ctx, lv.child.as_ref(), rm.as_ref(), cdt, keep || lv.ob > 0)?;
            if let Some(e) = deferred { return Err(e); }
            let offsets = if lv.ob > 0 { Some(offs.to_host((m + 1) * lv.ob)?) } else { None };
            Ok(rebuild(values, offsets, child, m, nulls_of(&validity, &o)?))
        }

        pub(super) fn child_take(ctx: &Context, child: &dyn Array, map: &dyn Array, cdt: i32, extend: bool) -> Result<ArrayRef, ArrowError> {
            match child.data_type() {
                DataType::List(_) | DataType::LargeList(_) | DataType::FixedSizeList(_, _) => take(ctx, child, map, cdt, 0, extend),
                DataType::Struct(_) | DataType::Union(_, _) => nested::take(ctx, child, map, cdt, 0, extend),
                DataType::Utf8 | DataType::Binary | DataType::LargeUtf8 | DataType::LargeBinary if extend => {
                    let ob = match kind_of(child.data_type())? { Kind::Bytes(ob) => ob, _ => unreachable!() };
                    let (v, ix) = (DeviceArray::upload(ctx, child, false)?, DeviceArray::upload(ctx, map, false)?);
                    let m = map.len();
                    let mut probe = ColumnOut::new(ctx, child.data_type(), m, 0)?;
                    let mut need = 0i64;
                    ctx.check(unsafe {
                        ffi::acu_take_bytes_extend(ctx.raw(), ob as i32, v.view().values, v.column.data, v.view(), ix.view(), cdt,
                                                   probe.out.array.values, std::ptr::null_mut(), 0, &mut need, &mut probe.out.array)
                    })?;
                    let mut out = ColumnOut::new(ctx, child.data_type(), m, need as usize)?;
                    ctx.check(unsafe {
                        ffi::acu_take_bytes_extend(ctx.raw(), ob as i32, v.view().values, v.column.data, v.view(), ix.view(), cdt,
                                                   out.out.array.values, out.out.data, out.out.data_capacity, &mut out.out.data_len,
                                                   &mut out.out.array)
                    })?;
                    out.finish(child.data_type())
                }
                DataType::FixedSizeBinary(_) if extend => Ok(keep_width0_rows(super::take(child, map, None)?, map.len())),
                _ => super::take(child, map, None),
            }
        }
    }

    // ---- Struct, sparse Union, dense Union (filter.rs:597-622, :1010-1054, take.rs:270-298, :334-382) -----------------
    /// A struct's columns go through filter / take of their own types and acu_filter_nulls / acu_take_nulls give its
    /// NullBuffer. acu_filter_union / acu_take_union give a union's type ids and, for a dense union, its new offsets and a
    /// child row map grouped by field; child f is then taken (take) or extended (filter: MutableArrayData, the child step of
    /// a list take) with its slice of the map.
    mod nested {
        use super::*;
        use arrow_array::types::{Int32Type, UInt64Type};
        use arrow_array::{new_empty_array, Array, StructArray, UnionArray};
        use super::list::nulls_of;
        use arrow_buffer::ScalarBuffer;
        use arrow_schema::UnionMode;

        /// filter / take of a child with a borrowed plan (the caller owns it)
        fn filter_child(ctx: &Context, plan: *mut ffi::acu_filter_plan, child: &dyn Array, child_step: Option<bool>) -> Result<ArrayRef, ArrowError> {
            match child.data_type() {
                DataType::List(_) | DataType::LargeList(_) | DataType::FixedSizeList(_, _) => list::filter(ctx, plan, child, child_step),
                DataType::Struct(_) | DataType::Union(_, _) => filter(ctx, plan, child, child_step),
                _ => {
                    let p = std::mem::ManuallyDrop::new(FilterPredicate { plan: Plan { ctx: ctx.clone(), raw: plan } });
                    let c = p.filter(child)?;
                    if child_step == Some(true) && c.nulls().map_or(false, |n| n.null_count() == 0) {
                        return Ok(make_array(unsafe { c.to_data().into_builder().nulls(None).build_unchecked() }));
                    }
                    Ok(c)
                }
            }
        }

        fn union_view(ctx: &Context, u: &UnionArray, ids: &[i8]) -> Result<(ffi::acu_union_array, Vec<DeviceBuffer>), ArrowError> {
            let t = DeviceBuffer::from_host(ctx, u.type_ids().inner().as_slice())?;
            let mut d = ffi::acu_union_array { mode: ffi::ACU_UNION_SPARSE, n_fields: ids.len() as i32, field_type_ids: ids.as_ptr(),
                                               type_ids: t.as_ptr() as *const i8, offsets: std::ptr::null(), len: u.len() as i64 };
            let mut bufs = vec![t];
            if let Some(o) = u.offsets() {
                let ob = DeviceBuffer::from_host(ctx, o.inner().as_slice())?;
                d.mode = ffi::ACU_UNION_DENSE;
                d.offsets = ob.as_ptr() as *const i32;
                bufs.push(ob);
            }
            Ok((d, bufs))
        }

        fn finish_union(u: &UnionArray, tids: &DeviceBuffer, offs: Option<&DeviceBuffer>, n: usize, children: Vec<ArrayRef>) -> Result<ArrayRef, ArrowError> {
            let DataType::Union(fields, _) = u.data_type() else { unreachable!() };
            let t = ScalarBuffer::<i8>::new(tids.to_host(n)?, 0, n);
            let o = match offs { Some(b) => Some(ScalarBuffer::<i32>::new(b.to_host(n * 4)?, 0, n)), None => None };
            Ok(Arc::new(unsafe { UnionArray::new_unchecked(fields.clone(), t, o, children) }))
        }

        fn map_slice(map: &DeviceBuffer, starts: &[i64], f: usize, n: usize) -> Result<ArrayRef, ArrowError> {
            let all = ScalarBuffer::<i32>::new(map.to_host(n * 4)?, 0, n);
            let (a, b) = (starts[f] as usize, starts[f + 1] as usize);
            Ok(Arc::new(PrimitiveArray::<Int32Type>::new(all.slice(a, b - a), None)))
        }

        pub(super) fn filter(ctx: &Context, plan: *mut ffi::acu_filter_plan, values: &dyn Array, child_step: Option<bool>) -> Result<ArrayRef, ArrowError> {
            let n = unsafe { ffi::acu_filter_plan_count(plan) } as usize;
            let strategy = unsafe { ffi::acu_filter_plan_strategy(plan) };
            if let Some(s) = values.as_any().downcast_ref::<StructArray>() {  // filter_struct: every column, then filter_nulls
                let cols = s.columns().iter().map(|c| filter_child(ctx, plan, c.as_ref(), child_step)).collect::<Result<Vec<_>, _>>()?;
                let nv = DeviceArray::upload(ctx, &BooleanArray::new(BooleanBuffer::new_set(s.len()), s.nulls().cloned()), false)?;
                let mut v = *nv.view();
                v.values = std::ptr::null();
                let validity = DeviceBuffer::allocate(ctx, bitmap_bytes(n.max(1)))?;
                let mut o = ffi::acu_array_out { values: std::ptr::null_mut(), validity: validity.as_ptr() as *mut u8, len: 0, null_count: 0, has_validity: 0, reserved: 0 };
                ctx.check(unsafe { ffi::acu_filter_nulls(ctx.raw(), plan, &v, &mut o) })?;
                if child_step == Some(true) && o.null_count == 0 { o.has_validity = 0; }
                let DataType::Struct(fields) = s.data_type() else { unreachable!() };
                return Ok(Arc::new(unsafe { StructArray::new_unchecked_with_length(fields.clone(), cols, nulls_of(&validity, &o)?, n) }));
            }
            let u = values.as_any().downcast_ref::<UnionArray>().unwrap();
            let DataType::Union(fields, mode) = u.data_type() else { unreachable!() };
            let dense = *mode == UnionMode::Dense;
            if dense && child_step == Some(true) && strategy == 1 {
                // a list's child step extends every row even when its plan selects them all: the rows of a take of 0 .. n
                let ids = PrimitiveArray::<UInt64Type>::from_iter_values(0..n as u64);
                return take(ctx, values, &ids, 7, 0, true);
            }
            let ids: Vec<i8> = fields.iter().map(|(t, _)| t).collect();
            let (d, _bufs) = union_view(ctx, u, &ids)?;
            let (tids, offs, map) = (DeviceBuffer::allocate(ctx, n.max(1))?, DeviceBuffer::allocate(ctx, n.max(1) * 4)?, DeviceBuffer::allocate(ctx, n.max(1) * 4)?);
            let mut starts = vec![0i64; ids.len() + 1];
            ctx.check(unsafe { ffi::acu_filter_union(ctx.raw(), plan, &d, tids.as_ptr() as *mut i8, offs.as_ptr() as *mut i32,
                                                     map.as_ptr() as *mut i32, starts.as_mut_ptr()) })?;
            if strategy == 1 { return Ok(u.slice(0, n)); }  // values.slice(0, count)
            if dense {
                let children = (0..ids.len()).map(|f| {
                    let rows = map_slice(&map, &starts, f, n)?;
                    list::child_take(ctx, u.child(ids[f]).as_ref(), rows.as_ref(), 2, true)  // ACU_I32, extended row by row
                }).collect::<Result<Vec<_>, _>>()?;
                return finish_union(u, &tids, Some(&offs), n, children);
            }
            let children = ids.iter().map(|&t| filter_child(ctx, plan, u.child(t).as_ref(), child_step)).collect::<Result<Vec<_>, _>>()?;
            if strategy == 0 { return Ok(new_empty_array(u.data_type())); }
            finish_union(u, &tids, None, n, children)
        }

        pub(super) fn take(ctx: &Context, values: &dyn Array, indices: &dyn Array, idt: i32, check: i32, keep: bool) -> Result<ArrayRef, ArrowError> {
            let ix = DeviceArray::upload(ctx, indices, false)?;
            let m = indices.len();
            let child_take = |child: &dyn Array, rows: &dyn Array, cdt: i32| list::child_take(ctx, child, rows, cdt, keep);
            if let Some(s) = values.as_any().downcast_ref::<StructArray>() {
                // take_impl's Struct arm: check_bounds first, then the columns, then the validity (its panic after theirs)
                let nv = DeviceArray::upload(ctx, &BooleanArray::new(BooleanBuffer::new_set(s.len()), s.nulls().cloned()), false)?;
                let mut v = *nv.view();
                v.values = std::ptr::null();
                let validity = DeviceBuffer::allocate(ctx, bitmap_bytes(m.max(1)))?;
                let mut o = ffi::acu_array_out { values: std::ptr::null_mut(), validity: validity.as_ptr() as *mut u8, len: 0, null_count: 0, has_validity: 0, reserved: 0 };
                let st = unsafe { ffi::acu_take_nulls(ctx.raw(), &v, ix.view(), idt, check, &mut o) };
                let deferred = if st == ffi::ACU_ERR_PANIC_OUT_OF_BOUNDS { Some(ctx.check(st).unwrap_err()) } else { ctx.check(st).map(|_| None)? };
                let cols = s.columns().iter().map(|c| child_take(c.as_ref(), indices, idt)).collect::<Result<Vec<_>, _>>()?;
                if let Some(e) = deferred { return Err(e); }
                let mut nulls = nulls_of(&validity, &o)?;
                if cols.is_empty() && !keep && nulls.is_none() { nulls = Some(NullBuffer::new_valid(m)); }  // new_empty_fields
                let DataType::Struct(fields) = s.data_type() else { unreachable!() };
                return Ok(Arc::new(unsafe { StructArray::new_unchecked_with_length(fields.clone(), cols, nulls, m) }));
            }
            let u = values.as_any().downcast_ref::<UnionArray>().unwrap();
            let DataType::Union(fields, mode) = u.data_type() else { unreachable!() };
            let dense = *mode == UnionMode::Dense;
            let ids: Vec<i8> = fields.iter().map(|(t, _)| t).collect();
            let (d, _bufs) = union_view(ctx, u, &ids)?;
            let (tids, offs, map) = (DeviceBuffer::allocate(ctx, m.max(1))?, DeviceBuffer::allocate(ctx, m.max(1) * 4)?, DeviceBuffer::allocate(ctx, m.max(1) * 4)?);
            let mut starts = vec![0i64; ids.len() + 1];
            let st = unsafe { ffi::acu_take_union(ctx.raw(), &d, ix.view(), idt, check, tids.as_ptr() as *mut i8, offs.as_ptr() as *mut i32,
                                                  map.as_ptr() as *mut i32, starts.as_mut_ptr()) };
            // UnionArray::try_new validates after the children are taken
            let deferred = match ctx.check(st) {
                Err(e) if e.to_string().ends_with("Type Ids values must match one of the field type ids")
                    || e.to_string().ends_with("Offsets must be non-negative and within the length of the Array") => Some(e),
                Err(e) => return Err(e),
                Ok(()) => None,
            };
            let children = (0..ids.len()).map(|f| {
                if dense { child_take(u.child(ids[f]).as_ref(), map_slice(&map, &starts, f, m)?.as_ref(), 2) }
                else { child_take(u.child(ids[f]).as_ref(), indices, idt) }
            }).collect::<Result<Vec<_>, _>>()?;
            if let Some(e) = deferred { return Err(e); }
            finish_union(u, &tids, if dense { Some(&offs) } else { None }, m, children)
        }
    }

    /// `arrow::compute::take_arrays` (take.rs:155-164).
    pub fn take_arrays(arrays: &[ArrayRef], indices: &dyn Array, options: Option<TakeOptions>) -> Result<Vec<ArrayRef>, ArrowError> {
        arrays.iter().map(|a| take(a.as_ref(), indices, options.clone())).collect()
    }
    /// `arrow::compute::take_record_batch` (take.rs:1123-1133).
    pub fn take_record_batch(record_batch: &RecordBatch, indices: &dyn Array) -> Result<RecordBatch, ArrowError> {
        let cols = take_arrays(record_batch.columns(), indices, None)?;
        RecordBatch::try_new(record_batch.schema(), cols)
    }

    // ---- cast (arrow-cast/src/cast/mod.rs) -----------------------------------------------------------------------------
    /// mod.rs:96-111 (format options are irrelevant to numeric casts)
    #[derive(Clone, Debug)]
    pub struct CastOptions { pub safe: bool }
    impl Default for CastOptions { fn default() -> Self { Self { safe: true } } }

    /// `arrow::compute::cast` (mod.rs:347-349).
    pub fn cast(array: &dyn Array, to_type: &DataType) -> Result<ArrayRef, ArrowError> { cast_with_options(array, to_type, &CastOptions::default()) }
    /// `arrow::compute::cast_with_options` (mod.rs:790): numeric -> numeric on the device; Dictionary<_, Utf8> -> Utf8 through take
    /// (arrow-cast/src/cast/dictionary.rs:310-317); any other pair is outside the hot path (SURVEY.md §8: out of scope).
    pub fn cast_with_options(array: &dyn Array, to_type: &DataType, options: &CastOptions) -> Result<ArrayRef, ArrowError> {
        if array.data_type() == to_type { return Ok(make_array(array.to_data())); }
        if let (DataType::Dictionary(_, v), DataType::Utf8) = (array.data_type(), to_type) {
            if **v == DataType::Utf8 {
                let d = array.to_data();
                let values = make_array(d.child_data()[0].clone());
                let keys = make_array(d.clone().into_builder().data_type(match array.data_type() { DataType::Dictionary(k, _) => (**k).clone(), _ => unreachable!() })
                    .child_data(vec![]).build()?);
                return take(values.as_ref(), keys.as_ref(), None);
            }
        }
        // the decimal arms (mod.rs:980-1219): decimal -> decimal, integer / float -> decimal, decimal -> integer / float
        let (from_dec, to_dec) = (decimal_type(array.data_type()), decimal_type(to_type));
        if from_dec.is_some() || to_dec.is_some() {
            let (fc, tc) = (dtype_code(array.data_type()), dtype_code(to_type));
            if !matches!((&from_dec, &to_dec, fc, tc), (Some(_), Some(_), _, _) | (None, Some(_), Some(_), _) | (Some(_), None, _, Some(_))) {
                return Err(ArrowError::CastError(format!("Casting from {} to {} not supported", array.data_type(), to_type)));
            }
            let ctx = Context::current()?;
            let a = DeviceArray::upload(&ctx, array, false)?;
            let mut out = ColumnOut::new(&ctx, to_type, array.len(), 0)?;
            let safe = options.safe as i32;
            let st = match (from_dec, to_dec) {
                (Some(f), Some(t)) => unsafe { ffi::acu_cast_decimal(ctx.raw(), &f, &t, safe, a.view(), out.array_out()) },
                (None, Some(t)) => unsafe { ffi::acu_cast_to_decimal(ctx.raw(), fc.unwrap(), &t, safe, a.view(), out.array_out()) },
                (Some(f), None) => unsafe { ffi::acu_cast_from_decimal(ctx.raw(), &f, tc.unwrap(), safe, a.view(), out.array_out()) },
                (None, None) => unreachable!(),
            };
            ctx.check(st)?;
            return out.finish(to_type);
        }
        let (from, to) = match (dtype_code(array.data_type()), dtype_code(to_type)) {
            (Some(f), Some(t)) => (f, t),
            _ => return Err(ArrowError::CastError(format!("Casting from {} to {} not supported", array.data_type(), to_type))),
        };
        let ctx = Context::current()?;
        let a = DeviceArray::upload(&ctx, array, false)?;
        let mut out = ColumnOut::new(&ctx, to_type, array.len(), 0)?;
        ctx.check(unsafe { ffi::acu_cast_numeric(ctx.raw(), from, to, options.safe as i32, a.view(), out.array_out()) })?;
        out.finish(to_type)
    }

    // ---- aggregate (arrow-arith/src/aggregate.rs) ------------------------------------------------------------------------
    fn aggregate<T: ArrowPrimitiveType>(op: i32, array: &PrimitiveArray<T>) -> Option<T::Native> {
        let dtype = native_code(&T::DATA_TYPE)?; // derived from T: a caller cannot pass a mismatching code
        let ctx = Context::current().ok()?;
        let a = DeviceArray::upload(&ctx, array, false).ok()?;
        let (mut bits, mut valid) = ([0u64; 2], 0i64);
        let st = if dtype == ffi::ACU_I128 { // Decimal128: sum wraps in i128, min / max in i128 order
            unsafe { ffi::acu_aggregate_i128(ctx.raw(), op, a.view(), bits.as_mut_ptr(), &mut valid) }
        } else {
            unsafe { ffi::acu_aggregate(ctx.raw(), dtype, op, a.view(), bits.as_mut_ptr(), &mut valid) }
        };
        ctx.check(st).ok()?;
        if valid == 0 { return None; }
        Some(unsafe { std::ptr::read_unaligned(bits.as_ptr() as *const T::Native) }) // native bit pattern, zero-extended, little endian
    }
    /// aggregate.rs:943 / :1012 / :1027 — `None` iff no valid row.
    pub fn sum<T: ArrowPrimitiveType>(array: &PrimitiveArray<T>) -> Option<T::Native> { aggregate(ffi::ACU_SUM, array) }
    pub fn min<T: ArrowPrimitiveType>(array: &PrimitiveArray<T>) -> Option<T::Native> { aggregate(ffi::ACU_MIN, array) }
    pub fn max<T: ArrowPrimitiveType>(array: &PrimitiveArray<T>) -> Option<T::Native> { aggregate(ffi::ACU_MAX, array) }
    /// aggregate.rs:953 (mul_wrapping for integers) and :850-875 (integer arrays only) — `None` iff no valid row.
    pub fn product<T: ArrowPrimitiveType>(array: &PrimitiveArray<T>) -> Option<T::Native> { aggregate(ffi::ACU_PRODUCT, array) }
    pub fn bit_and<T: ArrowPrimitiveType>(array: &PrimitiveArray<T>) -> Option<T::Native> { aggregate(ffi::ACU_BIT_AND, array) }
    pub fn bit_or<T: ArrowPrimitiveType>(array: &PrimitiveArray<T>) -> Option<T::Native> { aggregate(ffi::ACU_BIT_OR, array) }
    pub fn bit_xor<T: ArrowPrimitiveType>(array: &PrimitiveArray<T>) -> Option<T::Native> { aggregate(ffi::ACU_BIT_XOR, array) }
    type CheckedFold = unsafe extern "C" fn(*mut ffi::acu_ctx, i32, *const ffi::acu_array, *mut u64, *mut i64) -> ffi::acu_status;
    fn checked_fold<T: ArrowPrimitiveType>(f: CheckedFold, array: &PrimitiveArray<T>) -> Result<Option<T::Native>, ArrowError> {
        let dtype = numeric_dtype("arithmetic", &T::DATA_TYPE)?;
        let ctx = Context::current()?;
        let a = DeviceArray::upload(&ctx, array, false)?;
        let (mut bits, mut valid) = (0u64, 0i64);
        ctx.check(unsafe { f(ctx.raw(), dtype, a.view(), &mut bits, &mut valid) })?;
        Ok((valid != 0).then(|| unsafe { std::ptr::read_unaligned(&bits as *const u64 as *const T::Native) }))
    }
    /// aggregate.rs:897-937
    pub fn sum_checked<T: ArrowPrimitiveType>(array: &PrimitiveArray<T>) -> Result<Option<T::Native>, ArrowError> {
        checked_fold(ffi::acu_sum_checked, array)
    }
    /// aggregate.rs:963-1001: Err(ArithmeticOverflow) at the first valid row whose running product overflows
    pub fn product_checked<T: ArrowPrimitiveType>(array: &PrimitiveArray<T>) -> Result<Option<T::Native>, ArrowError> {
        checked_fold(ffi::acu_product_checked, array)
    }

    /// min / max of byte, view, fixed-size-binary and boolean arrays (aggregate.rs:372-568, :880-889). The device returns the
    /// lowest row holding the extremal value; the result borrows that row from the host array, as the reference's does.
    /// `arrow::compute::like` (arrow-string/src/like.rs:83-216): the haystack first; Utf8 / LargeUtf8 / Utf8View take all eight,
    /// Binary / LargeBinary / BinaryView contains / starts_with / ends_with. Dictionary operands are not accepted.
    pub mod like {
        use super::super::{ffi, ColumnOut, Context, DeviceArray, DeviceBuffer};
        use arrow_array::types::ByteViewType;
        use arrow_array::{Array, BooleanArray, Datum, GenericByteViewArray};
        use arrow_array::cast::AsArray;
        use arrow_schema::{ArrowError, DataType};

        const OP_NAMES: [&str; 8] = ["LIKE", "NLIKE", "ILIKE", "NILIKE", "CONTAINS", "STARTS_WITH", "ENDS_WITH", "EQ_IGNORE_ASCII_CASE"];

        fn view_operand<T: ByteViewType + ?Sized>(ctx: &Context, a: &GenericByteViewArray<T>, scalar: bool, bufs: &mut Vec<DeviceBuffer>,
                                                  ptrs: &mut Vec<*const u8>) -> Result<ffi::acu_view_array, ArrowError> {
            let (validity, validity_offset, null_count) = match a.nulls() {
                Some(n) => {
                    let b = DeviceBuffer::from_host(ctx, n.buffer().as_slice())?;
                    let p = b.as_ptr() as *const u8;
                    bufs.push(b);
                    (p, n.offset() as i64, n.null_count() as i64)
                }
                None => (std::ptr::null(), 0, 0),
            };
            let v = DeviceBuffer::from_host(ctx, a.views().inner().as_slice())?;
            let views = v.as_ptr();
            bufs.push(v);
            for d in a.data_buffers() {
                let b = DeviceBuffer::from_host(ctx, d.as_slice())?;
                ptrs.push(b.as_ptr() as *const u8);
                bufs.push(b);
            }
            let nulls = ffi::acu_array { values: std::ptr::null(), values_offset: 0, validity, validity_offset, len: a.len() as i64, null_count,
                                         is_scalar: scalar as i32, reserved: 0 };
            Ok(ffi::acu_view_array { views, buffers: ptrs.as_ptr(), n_buffers: ptrs.len() as i32, reserved: 0, nulls })
        }

        /// like_op (like.rs:218-296)
        fn like_op(op: i32, lhs: &dyn Datum, rhs: &dyn Datum) -> Result<BooleanArray, ArrowError> {
            use DataType::*;
            let (l, l_s) = lhs.get();
            let (r, r_s) = rhs.get();
            let ctx = Context::current()?;
            let n = if l_s { r.len() } else { l.len() };
            let mut out = ColumnOut::new(&ctx, &DataType::Boolean, n, 0)?;
            let is_utf8 = matches!(l.data_type(), Utf8 | LargeUtf8 | Utf8View) as i32;
            let st = match (l.data_type(), r.data_type()) {
                (Utf8, Utf8) | (LargeUtf8, LargeUtf8) | (Binary, Binary) | (LargeBinary, LargeBinary) => {
                    let ob = if matches!(l.data_type(), LargeUtf8 | LargeBinary) { 8 } else { 4 };
                    let (a, b) = (DeviceArray::upload(&ctx, l, l_s)?, DeviceArray::upload(&ctx, r, r_s)?);
                    let (x, y) = (ffi::acu_bytes_array { offsets: a.view().values, data: a.column.data, nulls: *a.view() },
                                  ffi::acu_bytes_array { offsets: b.view().values, data: b.column.data, nulls: *b.view() });
                    unsafe { ffi::acu_like_bytes(ctx.raw(), ob, is_utf8, op, &x, &y, out.array_out()) }
                }
                (Utf8View, Utf8View) | (BinaryView, BinaryView) => {
                    let (mut bufs, mut lp, mut rp) = (Vec::new(), Vec::new(), Vec::new());
                    let (x, y) = if is_utf8 != 0 {
                        (view_operand(&ctx, l.as_string_view(), l_s, &mut bufs, &mut lp)?, view_operand(&ctx, r.as_string_view(), r_s, &mut bufs, &mut rp)?)
                    } else {
                        (view_operand(&ctx, l.as_binary_view(), l_s, &mut bufs, &mut lp)?, view_operand(&ctx, r.as_binary_view(), r_s, &mut bufs, &mut rp)?)
                    };
                    unsafe { ffi::acu_like_byte_view(ctx.raw(), is_utf8, op, &x, &y, out.array_out()) }
                }
                (l_t, r_t) => {
                    return Err(ArrowError::InvalidArgumentError(format!("Invalid string/binary operation: {l_t} {} {r_t}", OP_NAMES[op as usize])))
                }
            };
            ctx.check(st)?;
            let r = out.finish(&DataType::Boolean)?;
            Ok(r.as_any().downcast_ref::<BooleanArray>().unwrap().clone())
        }
        pub fn like(left: &dyn Datum, right: &dyn Datum) -> Result<BooleanArray, ArrowError> { like_op(ffi::ACU_LIKE, left, right) }
        pub fn ilike(left: &dyn Datum, right: &dyn Datum) -> Result<BooleanArray, ArrowError> { like_op(ffi::ACU_ILIKE, left, right) }
        pub fn nlike(left: &dyn Datum, right: &dyn Datum) -> Result<BooleanArray, ArrowError> { like_op(ffi::ACU_NLIKE, left, right) }
        pub fn nilike(left: &dyn Datum, right: &dyn Datum) -> Result<BooleanArray, ArrowError> { like_op(ffi::ACU_NILIKE, left, right) }
        pub fn starts_with(left: &dyn Datum, right: &dyn Datum) -> Result<BooleanArray, ArrowError> { like_op(ffi::ACU_STARTS_WITH, left, right) }
        pub fn ends_with(left: &dyn Datum, right: &dyn Datum) -> Result<BooleanArray, ArrowError> { like_op(ffi::ACU_ENDS_WITH, left, right) }
        pub fn contains(left: &dyn Datum, right: &dyn Datum) -> Result<BooleanArray, ArrowError> { like_op(ffi::ACU_CONTAINS, left, right) }
        pub fn eq_ignore_ascii_case(left: &dyn Datum, right: &dyn Datum) -> Result<BooleanArray, ArrowError> {
            like_op(ffi::ACU_EQ_IGNORE_ASCII_CASE, left, right)
        }
    }

    /// `arrow::compute::{length, bit_length}` (arrow-string/src/length.rs:26-200) and `substring`, `substring_by_char`
    /// (arrow-string/src/substring.rs:73-251) on Utf8 / LargeUtf8 / Binary / LargeBinary, Utf8View / BinaryView and
    /// FixedSizeBinary (`substring_by_char`: Utf8 / LargeUtf8). A view result shares the input's data buffers (long values keep
    /// their buffer index with an advanced offset); the reference's builder copies them into new buffers, and the logical
    /// values are equal. Dictionary and run-end-encoded inputs are not accepted here: apply to their values.
    pub mod substring {
        use super::super::{ffi, kind_of, ColumnOut, Context, DeviceArray, DeviceBuffer, Kind};
        use arrow_array::cast::AsArray;
        use arrow_array::types::ByteViewType;
        use arrow_array::{make_array, Array, ArrayRef, GenericByteViewArray};
        use arrow_buffer::{BooleanBuffer, NullBuffer, ScalarBuffer};
        use arrow_data::ArrayData;
        use arrow_schema::{ArrowError, DataType};
        use std::sync::Arc;

        fn bytes_operand(a: &DeviceArray) -> ffi::acu_bytes_array {
            ffi::acu_bytes_array { offsets: a.view().values, data: a.column.data, nulls: *a.view() }
        }

        pub(super) fn view_operand<T: ByteViewType + ?Sized>(ctx: &Context, a: &GenericByteViewArray<T>, bufs: &mut Vec<DeviceBuffer>,
                                                  ptrs: &mut Vec<*const u8>) -> Result<ffi::acu_view_array, ArrowError> {
            let (validity, validity_offset, null_count) = match a.nulls() {
                Some(n) => {
                    let b = DeviceBuffer::from_host(ctx, n.buffer().as_slice())?;
                    let p = b.as_ptr() as *const u8;
                    bufs.push(b);
                    (p, n.offset() as i64, n.null_count() as i64)
                }
                None => (std::ptr::null(), 0, 0),
            };
            let v = DeviceBuffer::from_host(ctx, a.views().inner().as_slice())?;
            let views = v.as_ptr();
            bufs.push(v);
            for d in a.data_buffers() {
                let b = DeviceBuffer::from_host(ctx, d.as_slice())?;
                ptrs.push(b.as_ptr() as *const u8);
                bufs.push(b);
            }
            let nulls = ffi::acu_array { values: std::ptr::null(), values_offset: 0, validity, validity_offset, len: a.len() as i64, null_count,
                                         is_scalar: 0, reserved: 0 };
            Ok(ffi::acu_view_array { views, buffers: ptrs.as_ptr(), n_buffers: ptrs.len() as i32, reserved: 0, nulls })
        }

        pub(super) fn fsb_operand(ctx: &Context, a: &dyn Array, width: usize, bufs: &mut Vec<DeviceBuffer>) -> Result<ffi::acu_array, ArrowError> {
            let d = a.to_data();
            let (validity, validity_offset, null_count) = match d.nulls() {
                Some(n) => {
                    let b = DeviceBuffer::from_host(ctx, n.buffer().as_slice())?;
                    let p = b.as_ptr() as *const u8;
                    bufs.push(b);
                    (p, n.offset() as i64, n.null_count() as i64)
                }
                None => (std::ptr::null(), 0, 0),
            };
            let vals = DeviceBuffer::from_host(ctx, &d.buffers()[0].as_slice()[d.offset() * width..(d.offset() + d.len()) * width])?;
            let values = vals.as_ptr();
            bufs.push(vals);
            Ok(ffi::acu_array { values, values_offset: 0, validity, validity_offset, len: d.len() as i64, null_count, is_scalar: 0, reserved: 0 })
        }

        fn length_op(op: i32, array: &dyn Array) -> Result<ArrayRef, ArrowError> {
            use DataType::*;
            let ctx = Context::current()?;
            let out_type = if matches!(array.data_type(), LargeUtf8 | LargeBinary) { Int64 } else { Int32 };
            let mut out = ColumnOut::new(&ctx, &out_type, array.len(), 0)?;
            let st = match array.data_type() {
                Utf8 | LargeUtf8 | Binary | LargeBinary => {
                    let ob = if out_type == Int64 { 8 } else { 4 };
                    let a = DeviceArray::upload(&ctx, array, false)?;
                    unsafe { ffi::acu_length_bytes(ctx.raw(), ob, op, &bytes_operand(&a), out.array_out()) }
                }
                Utf8View | BinaryView => {
                    let (mut bufs, mut ptrs) = (Vec::new(), Vec::new());
                    let v = if array.data_type() == &Utf8View { view_operand(&ctx, array.as_string_view(), &mut bufs, &mut ptrs)? }
                            else { view_operand(&ctx, array.as_binary_view(), &mut bufs, &mut ptrs)? };
                    unsafe { ffi::acu_length_byte_view(ctx.raw(), op, &v, out.array_out()) }
                }
                FixedSizeBinary(w) => {
                    let mut bufs = Vec::new();
                    let a = fsb_operand(&ctx, array, *w as usize, &mut bufs)?;
                    unsafe { ffi::acu_length_fixed_size_binary(ctx.raw(), *w, op, &a, out.array_out()) }
                }
                other => {
                    let name = if op == ffi::ACU_LENGTH { "length" } else { "bit_length" };
                    return Err(ArrowError::ComputeError(format!("{name} not supported for {other:?}")));
                }
            };
            ctx.check(st)?;
            out.finish(&out_type)
        }
        pub fn length(array: &dyn Array) -> Result<ArrayRef, ArrowError> { length_op(ffi::ACU_LENGTH, array) }
        pub fn bit_length(array: &dyn Array) -> Result<ArrayRef, ArrowError> { length_op(ffi::ACU_BIT_LENGTH, array) }

        /// The two-phase byte-array call: offsets and the byte count, then the bytes into a buffer of exactly that size.
        fn two_phase(ctx: &Context, array: &dyn Array,
                     call: &dyn Fn(&ffi::acu_bytes_array, *mut std::os::raw::c_void, *mut u8, i64, &mut i64, &mut ffi::acu_array_out) -> i32)
                     -> Result<ArrayRef, ArrowError> {
            let a = DeviceArray::upload(ctx, array, false)?;
            let x = bytes_operand(&a);
            let mut sizing = ColumnOut::new(ctx, array.data_type(), array.len(), 0)?;
            let mut total = 0i64;
            ctx.check(call(&x, sizing.out.array.values, std::ptr::null_mut(), 0, &mut total, &mut sizing.out.array))?;
            let mut out = ColumnOut::new(ctx, array.data_type(), array.len(), total as usize)?;
            let (offs, data, cap) = (out.out.array.values, out.out.data, out.out.data_capacity);
            ctx.check(call(&x, offs, data, cap, &mut out.out.data_len, &mut out.out.array))?;
            out.finish(array.data_type())
        }

        fn view_substring<T: ByteViewType + ?Sized>(ctx: &Context, a: &GenericByteViewArray<T>, is_utf8: i32, start: i64, has_len: i32,
                                                    len: u64) -> Result<ArrayRef, ArrowError> {
            let (mut bufs, mut ptrs) = (Vec::new(), Vec::new());
            let v = view_operand(ctx, a, &mut bufs, &mut ptrs)?;
            let out_views = DeviceBuffer::allocate(ctx, a.len().max(1) * 16)?;
            let validity = DeviceBuffer::allocate(ctx, super::super::bitmap_bytes(a.len().max(1)))?;
            let mut o = ffi::acu_array_out { values: out_views.as_ptr(), validity: validity.as_ptr() as *mut u8, len: 0, null_count: 0,
                                             has_validity: 0, reserved: 0 };
            ctx.check(unsafe { ffi::acu_substring_byte_view(ctx.raw(), is_utf8, start, has_len, len, &v, out_views.as_ptr(), &mut o) })?;
            let n = a.len();
            let nulls = if o.has_validity != 0 {
                let bits = BooleanBuffer::new(validity.to_host(super::super::bitmap_bytes(n))?, 0, n);
                Some(unsafe { NullBuffer::new_unchecked(bits, o.null_count as usize) })
            } else { None };
            let views = ScalarBuffer::<u128>::new(out_views.to_host(n * 16)?, 0, n);
            // long results point into the input's buffers: the result keeps them
            Ok(Arc::new(unsafe { GenericByteViewArray::<T>::new_unchecked(views, a.data_buffers().to_vec(), nulls) }))
        }

        /// `substring(array, start, length)` (substring.rs:73-118).
        pub fn substring(array: &dyn Array, start: i64, length: Option<u64>) -> Result<ArrayRef, ArrowError> {
            use DataType::*;
            let ctx = Context::current()?;
            let (has_len, len) = (length.is_some() as i32, length.unwrap_or(0));
            match array.data_type() {
                Utf8 | LargeUtf8 | Binary | LargeBinary => {
                    let ob = match kind_of(array.data_type())? { Kind::Bytes(ob) => ob as i32, _ => unreachable!() };
                    let is_utf8 = matches!(array.data_type(), Utf8 | LargeUtf8) as i32;
                    let data_len = array.to_data().buffers()[1].len() as i64;
                    two_phase(&ctx, array, &|x, offs, data, cap, total, nulls| unsafe {
                        ffi::acu_substring_bytes(ctx.raw(), ob, is_utf8, start, has_len, len, x, data_len, offs, data, cap, total, nulls)
                    })
                }
                Utf8View => view_substring(&ctx, array.as_string_view(), 1, start, has_len, len),
                BinaryView => view_substring(&ctx, array.as_binary_view(), 0, start, has_len, len),
                FixedSizeBinary(w) => {
                    let mut bufs = Vec::new();
                    let a = fsb_operand(&ctx, array, *w as usize, &mut bufs)?;
                    let n = array.len();
                    let values = DeviceBuffer::allocate(&ctx, (n * *w as usize).max(1))?;
                    let validity = DeviceBuffer::allocate(&ctx, super::super::bitmap_bytes(n.max(1)))?;
                    let mut o = ffi::acu_array_out { values: values.as_ptr(), validity: validity.as_ptr() as *mut u8, len: 0, null_count: 0,
                                                     has_validity: 0, reserved: 0 };
                    let mut new_len = 0i32;
                    ctx.check(unsafe { ffi::acu_substring_fixed_size_binary(ctx.raw(), *w, start, has_len, len, &a, &mut new_len, &mut o) })?;
                    let nulls = if o.has_validity != 0 {
                        let bits = BooleanBuffer::new(validity.to_host(super::super::bitmap_bytes(n))?, 0, n);
                        Some(unsafe { NullBuffer::new_unchecked(bits, o.null_count as usize) })
                    } else { None };
                    let d = ArrayData::builder(FixedSizeBinary(new_len)).len(n).nulls(nulls)
                        .add_buffer(values.to_host(n * new_len as usize)?);
                    Ok(make_array(unsafe { d.build_unchecked() }))
                }
                other => Err(ArrowError::ComputeError(format!("substring does not support type {other:?}"))),
            }
        }

        /// `substring_by_char(array, start, length)` (substring.rs:144-165) for Utf8 / LargeUtf8.
        pub fn substring_by_char(array: &dyn Array, start: i64, length: Option<u64>) -> Result<ArrayRef, ArrowError> {
            let ctx = Context::current()?;
            let ob = match array.data_type() {
                DataType::Utf8 => 4,
                DataType::LargeUtf8 => 8,
                other => return Err(ArrowError::ComputeError(format!("substring_by_char does not support type {other:?}"))),
            };
            let (has_len, len) = (length.is_some() as i32, length.unwrap_or(0));
            two_phase(&ctx, array, &|x, offs, data, cap, total, nulls| unsafe {
                ffi::acu_substring_by_char(ctx.raw(), ob, start, has_len, len, x, offs, data, cap, total, nulls)
            })
        }
    }

    /// `arrow_string::concat_elements` (concat_elements.rs:31-476) on the device.
    pub mod concat_elements {
        use super::super::{ffi, ColumnOut, Context, DeviceArray, DeviceBuffer};
        use super::substring::{fsb_operand, view_operand};
        use arrow_array::cast::AsArray;
        use arrow_array::types::ByteViewType;
        use arrow_array::*;
        use arrow_buffer::{BooleanBuffer, Buffer, NullBuffer, ScalarBuffer};
        use arrow_data::ArrayData;
        use arrow_schema::{ArrowError, DataType};
        use std::sync::Arc;

        fn nulls_of(validity: &DeviceBuffer, o: &ffi::acu_array_out, n: usize) -> Result<Option<NullBuffer>, ArrowError> {
            if o.has_validity == 0 { return Ok(None); }
            let bits = BooleanBuffer::new(validity.to_host(super::super::bitmap_bytes(n))?, 0, n);
            Ok(Some(unsafe { NullBuffer::new_unchecked(bits, o.null_count as usize) }))
        }

        /// The two-phase byte-array call over `arrays` (one offset width): offsets and the byte count, then the bytes.
        fn bytes_many(arrays: &[&dyn Array]) -> Result<ArrayRef, ArrowError> {
            let ctx = Context::current()?;
            let dt = arrays.first().map(|a| a.data_type().clone()).unwrap_or(DataType::Utf8);
            let ob = if matches!(dt, DataType::LargeUtf8 | DataType::LargeBinary) { 8 } else { 4 };
            let uploaded = arrays.iter().map(|a| DeviceArray::upload(&ctx, *a, false)).collect::<Result<Vec<_>, _>>()?;
            let xs: Vec<ffi::acu_bytes_array> = uploaded.iter()
                .map(|a| ffi::acu_bytes_array { offsets: a.view().values, data: a.column.data, nulls: *a.view() }).collect();
            let n = arrays.first().map(|a| a.len()).unwrap_or(0);
            let mut sizing = ColumnOut::new(&ctx, &dt, n, 0)?;
            let mut total = 0i64;
            ctx.check(unsafe { ffi::acu_concat_elements_bytes_many(ctx.raw(), ob, xs.len() as i32, xs.as_ptr(), sizing.out.array.values,
                                                                   std::ptr::null_mut(), 0, &mut total, &mut sizing.out.array) })?;
            let mut out = ColumnOut::new(&ctx, &dt, n, total as usize)?;
            let (offs, data, cap) = (out.out.array.values, out.out.data, out.out.data_capacity);
            ctx.check(unsafe { ffi::acu_concat_elements_bytes_many(ctx.raw(), ob, xs.len() as i32, xs.as_ptr(), offs, data, cap,
                                                                   &mut out.out.data_len, &mut out.out.array) })?;
            out.finish(&dt)
        }

        fn check_len(l: usize, r: usize) -> Result<(), ArrowError> {
            if l != r { return Err(ArrowError::ComputeError(format!("Arrays must have the same length: {l} != {r}"))); }
            Ok(())
        }

        /// `concat_elements_bytes` (:31-75).
        pub fn concat_elements_bytes<T: types::ByteArrayType>(left: &GenericByteArray<T>, right: &GenericByteArray<T>)
                                                               -> Result<GenericByteArray<T>, ArrowError> {
            check_len(left.len(), right.len())?;
            Ok(bytes_many(&[left as &dyn Array, right as &dyn Array])?.as_bytes::<T>().clone())
        }
        /// `concat_elements_utf8` (:91-96).
        pub fn concat_elements_utf8<O: OffsetSizeTrait>(left: &GenericStringArray<O>, right: &GenericStringArray<O>)
                                                         -> Result<GenericStringArray<O>, ArrowError> {
            concat_elements_bytes(left, right)
        }
        /// `concat_element_binary` (:99-104).
        pub fn concat_element_binary<O: OffsetSizeTrait>(left: &GenericBinaryArray<O>, right: &GenericBinaryArray<O>)
                                                          -> Result<GenericBinaryArray<O>, ArrowError> {
            concat_elements_bytes(left, right)
        }
        /// `concat_elements_utf8_many` (:113-173).
        pub fn concat_elements_utf8_many<O: OffsetSizeTrait>(arrays: &[&GenericStringArray<O>]) -> Result<GenericStringArray<O>, ArrowError> {
            let dyns: Vec<&dyn Array> = arrays.iter().map(|a| *a as &dyn Array).collect();
            Ok(bytes_many(&dyns)?.as_string::<O>().clone())
        }

        /// `concat_elements_fixed_size_binary` (:181-228).
        pub fn concat_elements_fixed_size_binary(left: &FixedSizeBinaryArray, right: &FixedSizeBinaryArray)
                                                 -> Result<FixedSizeBinaryArray, ArrowError> {
            let ctx = Context::current()?;
            let (lw, rw) = (left.value_length(), right.value_length());
            let mut bufs = Vec::new();
            let l = fsb_operand(&ctx, left, lw.max(0) as usize, &mut bufs)?;
            let r = fsb_operand(&ctx, right, rw.max(0) as usize, &mut bufs)?;
            let n = left.len();
            let w = (lw.max(0) as usize) + (rw.max(0) as usize);
            let values = DeviceBuffer::allocate(&ctx, (n * w).max(1))?;
            let validity = DeviceBuffer::allocate(&ctx, super::super::bitmap_bytes(n.max(1)))?;
            let mut o = ffi::acu_array_out { values: values.as_ptr(), validity: validity.as_ptr() as *mut u8, len: 0, null_count: 0,
                                             has_validity: 0, reserved: 0 };
            let mut width = 0i32;
            ctx.check(unsafe { ffi::acu_concat_elements_fixed_size_binary(ctx.raw(), lw, &l, rw, &r, &mut width, &mut o) })?;
            let d = ArrayData::builder(DataType::FixedSizeBinary(width)).len(n).nulls(nulls_of(&validity, &o, n)?)
                .add_buffer(values.to_host(n * width as usize)?);
            Ok(FixedSizeBinaryArray::from(unsafe { d.build_unchecked() }))
        }

        fn view_concat<T: ByteViewType + ?Sized>(left: &GenericByteViewArray<T>, right: &GenericByteViewArray<T>)
                                                 -> Result<GenericByteViewArray<T>, ArrowError> {
            let ctx = Context::current()?;
            let (mut bufs, mut lp, mut rp) = (Vec::new(), Vec::new(), Vec::new());
            let l = view_operand(&ctx, left, &mut bufs, &mut lp)?;
            let r = view_operand(&ctx, right, &mut bufs, &mut rp)?;
            let n = left.len();
            let validity = DeviceBuffer::allocate(&ctx, super::super::bitmap_bytes(n.max(1)))?;
            let mut o = ffi::acu_array_out { values: std::ptr::null_mut(), validity: validity.as_ptr() as *mut u8, len: 0, null_count: 0,
                                             has_validity: 0, reserved: 0 };
            let mut total = 0i64;
            ctx.check(unsafe { ffi::acu_concat_elements_byte_view(ctx.raw(), &l, &r, std::ptr::null_mut(), std::ptr::null_mut(), 0, &mut total,
                                                                  &mut o) })?;
            let views = DeviceBuffer::allocate(&ctx, n.max(1) * 16)?;
            let data = DeviceBuffer::allocate(&ctx, (total as usize).max(1))?;
            ctx.check(unsafe { ffi::acu_concat_elements_byte_view(ctx.raw(), &l, &r, views.as_ptr(), data.as_ptr() as *mut u8, total, &mut total,
                                                                  &mut o) })?;
            let v = ScalarBuffer::<u128>::new(views.to_host(n * 16)?, 0, n);
            let buffers: Vec<Buffer> = if total > 0 { vec![data.to_host(total as usize)?] } else { vec![] };
            Ok(unsafe { GenericByteViewArray::<T>::new_unchecked(v, buffers, nulls_of(&validity, &o, n)?) })
        }
        /// `concat_elements_binary_view_array` (:388-393).
        pub fn concat_elements_binary_view_array(left: &BinaryViewArray, right: &BinaryViewArray) -> Result<BinaryViewArray, ArrowError> {
            view_concat(left, right)
        }
        /// `concat_elements_string_view_array` (:402-407).
        pub fn concat_elements_string_view_array(left: &StringViewArray, right: &StringViewArray) -> Result<StringViewArray, ArrowError> {
            view_concat(left, right)
        }

        /// `concat_elements_dyn` (:419-476).
        pub fn concat_elements_dyn(left: &dyn Array, right: &dyn Array) -> Result<ArrayRef, ArrowError> {
            use DataType::*;
            match (left.data_type(), right.data_type()) {
                (Utf8, Utf8) => Ok(Arc::new(concat_elements_utf8(left.as_string::<i32>(), right.as_string::<i32>())?)),
                (LargeUtf8, LargeUtf8) => Ok(Arc::new(concat_elements_utf8(left.as_string::<i64>(), right.as_string::<i64>())?)),
                (Binary, Binary) => Ok(Arc::new(concat_element_binary(left.as_binary::<i32>(), right.as_binary::<i32>())?)),
                (LargeBinary, LargeBinary) => Ok(Arc::new(concat_element_binary(left.as_binary::<i64>(), right.as_binary::<i64>())?)),
                (Utf8View, Utf8View) => Ok(Arc::new(concat_elements_string_view_array(left.as_string_view(), right.as_string_view())?)),
                (BinaryView, BinaryView) => Ok(Arc::new(concat_elements_binary_view_array(left.as_binary_view(), right.as_binary_view())?)),
                (FixedSizeBinary(_), FixedSizeBinary(_)) => {
                    Ok(Arc::new(concat_elements_fixed_size_binary(left.as_fixed_size_binary(), right.as_fixed_size_binary())?))
                }
                (l, r) if l != r => Err(ArrowError::ComputeError(format!("Cannot concat arrays of different types: {l} != {r}"))),
                (l, _) => Err(ArrowError::NotYetImplemented(format!("concat not supported for {l}"))),
            }
        }
    }

    pub mod aggregate {
        use super::super::{ffi, Context, DeviceArray, DeviceBuffer};
        use arrow_array::types::{BinaryViewType, ByteViewType, StringViewType};
        use arrow_array::{Array, BooleanArray, FixedSizeBinaryArray, GenericBinaryArray, GenericByteViewArray, GenericStringArray, OffsetSizeTrait};
        use arrow_schema::ArrowError;

        fn nulls_view(ctx: &Context, array: &dyn Array, bufs: &mut Vec<DeviceBuffer>) -> Result<ffi::acu_array, ArrowError> {
            let (validity, validity_offset, null_count) = match array.nulls() {
                Some(n) => {
                    let b = DeviceBuffer::from_host(ctx, n.buffer().as_slice())?;
                    let p = b.as_ptr() as *const u8;
                    bufs.push(b);
                    (p, n.offset() as i64, n.null_count() as i64)
                }
                None => (std::ptr::null(), 0, 0),
            };
            Ok(ffi::acu_array { values: std::ptr::null(), values_offset: 0, validity, validity_offset, len: array.len() as i64, null_count,
                                is_scalar: 0, reserved: 0 })
        }
        fn bytes_row<O: OffsetSizeTrait>(op: i32, array: &dyn Array) -> Option<usize> {
            let ctx = Context::current().ok()?;
            let a = DeviceArray::upload(&ctx, array, false).ok()?;
            let b = ffi::acu_bytes_array { offsets: a.column.array.values, data: a.column.data, nulls: a.column.array };
            let (mut row, mut valid) = (-1i64, 0i64);
            ctx.check(unsafe { ffi::acu_aggregate_bytes(ctx.raw(), std::mem::size_of::<O>() as i32, op, &b, &mut row, &mut valid) }).ok()?;
            (row >= 0).then_some(row as usize)
        }
        fn view_row<T: ByteViewType + ?Sized>(op: i32, array: &GenericByteViewArray<T>) -> Option<usize> {
            let ctx = Context::current().ok()?;
            let mut bufs = Vec::new();
            let nulls = nulls_view(&ctx, array, &mut bufs).ok()?;
            let views = array.views();
            let v = DeviceBuffer::from_host(&ctx, views.inner().as_slice()).ok()?;
            let views_ptr = v.as_ptr();
            bufs.push(v);
            let mut ptrs = Vec::new();
            for d in array.data_buffers() {
                let b = DeviceBuffer::from_host(&ctx, d.as_slice()).ok()?;
                ptrs.push(b.as_ptr() as *const u8);
                bufs.push(b);
            }
            let a = ffi::acu_view_array { views: views_ptr, buffers: ptrs.as_ptr(), n_buffers: ptrs.len() as i32, reserved: 0, nulls };
            let (mut row, mut valid) = (-1i64, 0i64);
            ctx.check(unsafe { ffi::acu_aggregate_byte_view(ctx.raw(), op, &a, &mut row, &mut valid) }).ok()?;
            (row >= 0).then_some(row as usize)
        }
        fn fixed_row(op: i32, array: &FixedSizeBinaryArray) -> Option<usize> {
            let ctx = Context::current().ok()?;
            let mut bufs = Vec::new();
            let mut a = nulls_view(&ctx, array, &mut bufs).ok()?;
            let w = array.value_length() as usize;
            let d = array.to_data();
            let bytes = &d.buffers()[0].as_slice()[d.offset() * w..(d.offset() + d.len()) * w];
            let v = DeviceBuffer::from_host(&ctx, bytes).ok()?;
            a.values = v.as_ptr();
            bufs.push(v);
            let (mut row, mut valid) = (-1i64, 0i64);
            ctx.check(unsafe { ffi::acu_aggregate_fixed_size_binary(ctx.raw(), w as i32, op, &a, &mut row, &mut valid) }).ok()?;
            (row >= 0).then_some(row as usize)
        }
        fn boolean(op: i32, array: &BooleanArray) -> Option<bool> {
            let ctx = Context::current().ok()?;
            let a = DeviceArray::upload(&ctx, array, false).ok()?;
            let (mut value, mut valid) = (-1i32, 0i64);
            ctx.check(unsafe { ffi::acu_aggregate_boolean(ctx.raw(), op, &a.column.array, &mut value, &mut valid) }).ok()?;
            (value >= 0).then_some(value != 0)
        }

        /// aggregate.rs:520-568
        pub fn max_binary<T: OffsetSizeTrait>(array: &GenericBinaryArray<T>) -> Option<&[u8]> { bytes_row::<T>(ffi::ACU_MAX, array).map(|i| array.value(i)) }
        pub fn min_binary<T: OffsetSizeTrait>(array: &GenericBinaryArray<T>) -> Option<&[u8]> { bytes_row::<T>(ffi::ACU_MIN, array).map(|i| array.value(i)) }
        pub fn max_string<T: OffsetSizeTrait>(array: &GenericStringArray<T>) -> Option<&str> { bytes_row::<T>(ffi::ACU_MAX, array).map(|i| array.value(i)) }
        pub fn min_string<T: OffsetSizeTrait>(array: &GenericStringArray<T>) -> Option<&str> { bytes_row::<T>(ffi::ACU_MIN, array).map(|i| array.value(i)) }
        pub fn max_binary_view(array: &GenericByteViewArray<BinaryViewType>) -> Option<&[u8]> { view_row(ffi::ACU_MAX, array).map(|i| array.value(i)) }
        pub fn min_binary_view(array: &GenericByteViewArray<BinaryViewType>) -> Option<&[u8]> { view_row(ffi::ACU_MIN, array).map(|i| array.value(i)) }
        pub fn max_string_view(array: &GenericByteViewArray<StringViewType>) -> Option<&str> { view_row(ffi::ACU_MAX, array).map(|i| array.value(i)) }
        pub fn min_string_view(array: &GenericByteViewArray<StringViewType>) -> Option<&str> { view_row(ffi::ACU_MIN, array).map(|i| array.value(i)) }
        pub fn max_fixed_size_binary(array: &FixedSizeBinaryArray) -> Option<&[u8]> { fixed_row(ffi::ACU_MAX, array).map(|i| array.value(i)) }
        pub fn min_fixed_size_binary(array: &FixedSizeBinaryArray) -> Option<&[u8]> { fixed_row(ffi::ACU_MIN, array).map(|i| array.value(i)) }
        /// aggregate.rs:372-457, :880-889
        pub fn min_boolean(array: &BooleanArray) -> Option<bool> { boolean(ffi::ACU_MIN, array) }
        pub fn max_boolean(array: &BooleanArray) -> Option<bool> { boolean(ffi::ACU_MAX, array) }
        pub fn bool_and(array: &BooleanArray) -> Option<bool> { min_boolean(array) }
        pub fn bool_or(array: &BooleanArray) -> Option<bool> { max_boolean(array) }
    }

    // ---- nullif / zip / concat (arrow-select) ----------------------------------------------------------------------------
    /// `arrow::compute::nullif` (nullif.rs:44): values shared, validity &= !(right is Some(true)).
    pub fn nullif(left: &dyn Array, right: &BooleanArray) -> Result<ArrayRef, ArrowError> {
        let ctx = Context::current()?;
        let (l, r) = (DeviceArray::upload(&ctx, left, false)?, DeviceArray::upload(&ctx, right, false)?);
        let validity = DeviceBuffer::allocate(&ctx, bitmap_bytes(left.len().max(1)))?;
        let mut out = ffi::acu_array_out { values: std::ptr::null_mut(), validity: validity.as_ptr() as *mut u8, len: 0, null_count: 0, has_validity: 0, reserved: 0 };
        ctx.check(unsafe { ffi::acu_nullif(ctx.raw(), l.view(), r.view(), &mut out) })?;
        if left.is_empty() { return Ok(make_array(left.to_data())); }
        let nulls = if out.has_validity != 0 {
            Some(unsafe { NullBuffer::new_unchecked(BooleanBuffer::new(validity.to_host(bitmap_bytes(left.len()))?, 0, left.len()), out.null_count as usize) })
        } else { None };
        // only the null mask changes; the host value buffers are shared (nullif.rs:107-112). The slice is normalised to
        // offset 0 first because the new mask has bit offset 0.
        let d = left.to_data();
        let d = if d.offset() != 0 {
            let mut m = arrow_data::transform::MutableArrayData::new(vec![&d], false, d.len());
            m.extend(0, 0, d.len());
            m.freeze()
        } else { d };
        Ok(make_array(unsafe { d.into_builder().nulls(nulls).build_unchecked() }))
    }

    /// `arrow::compute::zip` (zip.rs:99) for primitive arrays / scalars.
    pub fn zip(mask: &BooleanArray, truthy: &dyn Datum, falsy: &dyn Datum) -> Result<ArrayRef, ArrowError> {
        let (t, t_s) = truthy.get();
        let (f, f_s) = falsy.get();
        if t.data_type() != f.data_type() { return Err(ArrowError::InvalidArgumentError("arguments need to have the same data type".into())); }
        let w = t.data_type().primitive_width().ok_or_else(|| ArrowError::NotYetImplemented(format!("arrow-cuda zip: {}", t.data_type())))?;
        let ctx = Context::current()?;
        let (m, tv, fv) = (DeviceArray::upload(&ctx, mask, false)?, DeviceArray::upload(&ctx, t, t_s)?, DeviceArray::upload(&ctx, f, f_s)?);
        let mut out = ColumnOut::new(&ctx, t.data_type(), mask.len(), 0)?;
        ctx.check(unsafe { ffi::acu_zip(ctx.raw(), w as i32, m.view(), tv.view(), fv.view(), out.array_out()) })?;
        out.finish(t.data_type())
    }

    /// `arrow::compute::concat` (concat.rs:495).
    pub fn concat(arrays: &[&dyn Array]) -> Result<ArrayRef, ArrowError> {
        if arrays.is_empty() { return Err(ArrowError::ComputeError("concat requires input of at least one array".into())); }
        if arrays.len() == 1 { return Ok(arrays[0].slice(0, arrays[0].len())); }
        let d = arrays[0].data_type();
        if arrays.iter().skip(1).any(|a| a.data_type() != d) { // the reference lists up to 10 distinct types (concat.rs:505-535)
            let mut seen: Vec<&DataType> = vec![d];
            let mut msg = format!("It is not possible to concatenate arrays of different data types ({d}");
            for a in arrays {
                if !seen.contains(&a.data_type()) {
                    seen.push(a.data_type());
                    if seen.len() == 11 { msg.push_str(", ..."); break; }
                    msg.push_str(", ");
                    msg.push_str(&a.data_type().to_string());
                }
            }
            msg.push_str(").");
            return Err(ArrowError::InvalidArgumentError(msg));
        }
        let ctx = Context::current()?;
        let ups = arrays.iter().map(|a| DeviceArray::upload(&ctx, *a, false)).collect::<Result<Vec<_>, _>>()?;
        let cols: Vec<ffi::acu_column> = ups.iter().map(|u| u.column).collect();
        let rows: usize = arrays.iter().map(|a| a.len()).sum();
        let mut out = ColumnOut::new(&ctx, d, rows, ups.iter().map(|u| u.data_bytes).sum())?;
        ctx.check(unsafe { ffi::acu_concat(ctx.raw(), cols.len() as i32, cols.as_ptr(), &mut out.out) })?;
        out.finish(d)
    }
    /// `arrow::compute::concat_batches` (concat.rs:607).
    pub fn concat_batches<'a>(schema: &SchemaRef, input_batches: impl IntoIterator<Item = &'a RecordBatch>) -> Result<RecordBatch, ArrowError> {
        let batches: Vec<&RecordBatch> = input_batches.into_iter().collect();
        if schema.fields().is_empty() {
            let rows = batches.iter().map(|b| b.num_rows()).sum();
            return RecordBatch::try_new_with_options(schema.clone(), vec![], &arrow_array::RecordBatchOptions::new().with_row_count(Some(rows)));
        }
        if batches.is_empty() { return Ok(RecordBatch::new_empty(schema.clone())); }
        let cols = (0..schema.fields().len())
            .map(|i| concat(&batches.iter().map(|b| b.column(i).as_ref()).collect::<Vec<_>>()))
            .collect::<Result<Vec<_>, _>>()?;
        RecordBatch::try_new(schema.clone(), cols)
    }

    // ---- kernels ------------------------------------------------------------------------------------------------------------
    pub mod kernels {
        use super::*;

        /// `arrow::compute::kernels::numeric` (arrow-arith/src/numeric.rs:36-186)
        pub mod numeric {
            use super::*;
            /// decimal_op (numeric.rs:970-1107): the result DataType comes back from the device call
            fn decimal_op(op: i32, l: &dyn Array, l_s: bool, r: &dyn Array, r_s: bool) -> Result<ArrayRef, ArrowError> {
                let (lt, rt) = (decimal_type(l.data_type()).unwrap(), decimal_type(r.data_type()).unwrap());
                let ctx = Context::current()?;
                let (a, b) = (DeviceArray::upload(&ctx, l, l_s)?, DeviceArray::upload(&ctx, r, r_s)?);
                let n = if l_s && !r_s { r.len() } else { l.len() };
                let mut out = ColumnOut::new(&ctx, l.data_type(), n, 0)?;
                let mut ot = ffi::acu_decimal_type::default();
                ctx.check(unsafe { ffi::acu_decimal_arith(ctx.raw(), op, &lt, a.view(), &rt, b.view(), &mut ot, out.array_out()) })?;
                out.finish(&match ot.byte_width {
                    4 => DataType::Decimal32(ot.precision, ot.scale),
                    8 => DataType::Decimal64(ot.precision, ot.scale),
                    _ => DataType::Decimal128(ot.precision, ot.scale),
                })
            }
            fn arithmetic_op(op: i32, sym: &str, lhs: &dyn Datum, rhs: &dyn Datum) -> Result<ArrayRef, ArrowError> {
                let (l, l_s) = lhs.get();
                let (r, r_s) = rhs.get();
                match (l.data_type(), r.data_type()) { // the (Decimal*, Decimal*) arms of numeric.rs:257-259
                    (DataType::Decimal32(_, _), DataType::Decimal32(_, _))
                    | (DataType::Decimal64(_, _), DataType::Decimal64(_, _))
                    | (DataType::Decimal128(_, _), DataType::Decimal128(_, _)) => return decimal_op(op, l, l_s, r, r_s),
                    _ => {}
                }
                let dtype = match (dtype_code(l.data_type()), l.data_type() == r.data_type()) { // numeric.rs:270-272
                    (Some(c), true) => c,
                    _ => return Err(ArrowError::InvalidArgumentError(format!("Invalid arithmetic operation: {} {sym} {}", l.data_type(), r.data_type()))),
                };
                let ctx = Context::current()?;
                let (a, b) = (DeviceArray::upload(&ctx, l, l_s)?, DeviceArray::upload(&ctx, r, r_s)?);
                let n = if l_s && !r_s { r.len() } else { l.len() };
                let mut out = ColumnOut::new(&ctx, l.data_type(), n, 0)?;
                ctx.check(unsafe { ffi::acu_arith(ctx.raw(), dtype, op, a.view(), b.view(), out.array_out()) })?;
                out.finish(l.data_type())
            }
            pub fn add(lhs: &dyn Datum, rhs: &dyn Datum) -> Result<ArrayRef, ArrowError> { arithmetic_op(ffi::ACU_ADD, "+", lhs, rhs) }
            pub fn add_wrapping(lhs: &dyn Datum, rhs: &dyn Datum) -> Result<ArrayRef, ArrowError> { arithmetic_op(ffi::ACU_ADD_WRAPPING, "+", lhs, rhs) }
            pub fn sub(lhs: &dyn Datum, rhs: &dyn Datum) -> Result<ArrayRef, ArrowError> { arithmetic_op(ffi::ACU_SUB, "-", lhs, rhs) }
            pub fn sub_wrapping(lhs: &dyn Datum, rhs: &dyn Datum) -> Result<ArrayRef, ArrowError> { arithmetic_op(ffi::ACU_SUB_WRAPPING, "-", lhs, rhs) }
            pub fn mul(lhs: &dyn Datum, rhs: &dyn Datum) -> Result<ArrayRef, ArrowError> { arithmetic_op(ffi::ACU_MUL, "*", lhs, rhs) }
            pub fn mul_wrapping(lhs: &dyn Datum, rhs: &dyn Datum) -> Result<ArrayRef, ArrowError> { arithmetic_op(ffi::ACU_MUL_WRAPPING, "*", lhs, rhs) }
            pub fn div(lhs: &dyn Datum, rhs: &dyn Datum) -> Result<ArrayRef, ArrowError> { arithmetic_op(ffi::ACU_DIV, "/", lhs, rhs) }
            pub fn rem(lhs: &dyn Datum, rhs: &dyn Datum) -> Result<ArrayRef, ArrowError> { arithmetic_op(ffi::ACU_REM, "%", lhs, rhs) }
            fn neg_op(array: &dyn Array, checked: i32) -> Result<ArrayRef, ArrowError> {
                // decimals: neg_checked at every width (numeric.rs:116-136); neg_wrapping falls back to neg (:181-186)
                let (dtype, checked) = match (decimal_type(array.data_type()), native_code(array.data_type())) {
                    (Some(_), Some(code)) => (code, 1),
                    _ => (numeric_dtype("arithmetic", array.data_type())?, checked),
                };
                let ctx = Context::current()?;
                let a = DeviceArray::upload(&ctx, array, false)?;
                let mut out = ColumnOut::new(&ctx, array.data_type(), array.len(), 0)?;
                ctx.check(unsafe { ffi::acu_neg(ctx.raw(), dtype, checked, a.view(), out.array_out()) })?;
                out.finish(array.data_type())
            }
            pub fn neg(array: &dyn Array) -> Result<ArrayRef, ArrowError> { neg_op(array, 1) }
            pub fn neg_wrapping(array: &dyn Array) -> Result<ArrayRef, ArrowError> { neg_op(array, 0) }
        }

        /// `arrow::compute::kernels::cmp` (arrow-ord/src/cmp.rs:79-202)
        pub mod cmp {
            use super::*;
            fn compare_op(op: i32, sym: &str, lhs: &dyn Datum, rhs: &dyn Datum) -> Result<BooleanArray, ArrowError> {
                let (l, l_s) = lhs.get();
                let (r, r_s) = rhs.get();
                if l.data_type() != r.data_type() { // cmp.rs:260-264
                    return Err(ArrowError::InvalidArgumentError(format!("Invalid comparison operation: {} {sym} {}", l.data_type(), r.data_type())));
                }
                let ctx = Context::current()?;
                let (a, b) = (DeviceArray::upload(&ctx, l, l_s)?, DeviceArray::upload(&ctx, r, r_s)?);
                let n = if l_s { r.len() } else { l.len() };
                let mut out = ColumnOut::new(&ctx, &DataType::Boolean, n, 0)?;
                let st = match kind_of(l.data_type())? {
                    Kind::FixedSizeBinary(_) => return Err(ArrowError::NotYetImplemented(format!("arrow-cuda: data type {}", l.data_type()))),
                    Kind::Bytes(ob) => {
                        let (x, y) = (ffi::acu_bytes_array { offsets: a.view().values, data: a.column.data, nulls: *a.view() },
                                      ffi::acu_bytes_array { offsets: b.view().values, data: b.column.data, nulls: *b.view() });
                        unsafe { ffi::acu_cmp_bytes(ctx.raw(), ob as i32, op, &x, &y, out.array_out()) }
                    }
                    _ => {
                        let dtype = native_code(l.data_type()) // decimals compare as their natives
                            .ok_or_else(|| ArrowError::InvalidArgumentError(format!("Invalid comparison operation: {} {sym} {}", l.data_type(), r.data_type())))?;
                        unsafe { ffi::acu_cmp(ctx.raw(), dtype, op, a.view(), b.view(), out.array_out()) }
                    }
                };
                ctx.check(st)?;
                let r = out.finish(&DataType::Boolean)?;
                Ok(r.as_any().downcast_ref::<BooleanArray>().unwrap().clone())
            }
            pub fn eq(lhs: &dyn Datum, rhs: &dyn Datum) -> Result<BooleanArray, ArrowError> { compare_op(ffi::ACU_EQ, "==", lhs, rhs) }
            pub fn neq(lhs: &dyn Datum, rhs: &dyn Datum) -> Result<BooleanArray, ArrowError> { compare_op(ffi::ACU_NEQ, "!=", lhs, rhs) }
            pub fn lt(lhs: &dyn Datum, rhs: &dyn Datum) -> Result<BooleanArray, ArrowError> { compare_op(ffi::ACU_LT, "<", lhs, rhs) }
            pub fn lt_eq(lhs: &dyn Datum, rhs: &dyn Datum) -> Result<BooleanArray, ArrowError> { compare_op(ffi::ACU_LT_EQ, "<=", lhs, rhs) }
            pub fn gt(lhs: &dyn Datum, rhs: &dyn Datum) -> Result<BooleanArray, ArrowError> { compare_op(ffi::ACU_GT, ">", lhs, rhs) }
            pub fn gt_eq(lhs: &dyn Datum, rhs: &dyn Datum) -> Result<BooleanArray, ArrowError> { compare_op(ffi::ACU_GT_EQ, ">=", lhs, rhs) }
            pub fn distinct(lhs: &dyn Datum, rhs: &dyn Datum) -> Result<BooleanArray, ArrowError> { compare_op(ffi::ACU_DISTINCT, "IS DISTINCT FROM", lhs, rhs) }
            pub fn not_distinct(lhs: &dyn Datum, rhs: &dyn Datum) -> Result<BooleanArray, ArrowError> { compare_op(ffi::ACU_NOT_DISTINCT, "IS NOT DISTINCT FROM", lhs, rhs) }
        }

        /// `arrow::compute::kernels::boolean` (arrow-arith/src/boolean.rs:60-354)
        pub mod boolean {
            use super::*;
            fn boolean_op(op: i32, a: &dyn Array, b: Option<&BooleanArray>) -> Result<BooleanArray, ArrowError> {
                let ctx = Context::current()?;
                let da = DeviceArray::upload(&ctx, a, false)?;
                let db = b.map(|b| DeviceArray::upload(&ctx, b, false)).transpose()?;
                let mut out = ColumnOut::new(&ctx, &DataType::Boolean, a.len(), 0)?;
                ctx.check(unsafe { ffi::acu_boolean(ctx.raw(), op, da.view(), db.as_ref().map_or(std::ptr::null(), |d| d.view() as *const _), out.array_out()) })?;
                Ok(out.finish(&DataType::Boolean)?.as_any().downcast_ref::<BooleanArray>().unwrap().clone())
            }
            pub fn and(left: &BooleanArray, right: &BooleanArray) -> Result<BooleanArray, ArrowError> { boolean_op(ffi::ACU_BOOL_AND, left, Some(right)) }
            pub fn or(left: &BooleanArray, right: &BooleanArray) -> Result<BooleanArray, ArrowError> { boolean_op(ffi::ACU_BOOL_OR, left, Some(right)) }
            pub fn and_not(left: &BooleanArray, right: &BooleanArray) -> Result<BooleanArray, ArrowError> { boolean_op(ffi::ACU_BOOL_AND_NOT, left, Some(right)) }
            pub fn and_kleene(left: &BooleanArray, right: &BooleanArray) -> Result<BooleanArray, ArrowError> { boolean_op(ffi::ACU_BOOL_AND_KLEENE, left, Some(right)) }
            pub fn or_kleene(left: &BooleanArray, right: &BooleanArray) -> Result<BooleanArray, ArrowError> { boolean_op(ffi::ACU_BOOL_OR_KLEENE, left, Some(right)) }
            pub fn not(left: &BooleanArray) -> Result<BooleanArray, ArrowError> { boolean_op(ffi::ACU_BOOL_NOT, left, None) }
            pub fn is_null(input: &dyn Array) -> Result<BooleanArray, ArrowError> { boolean_op(ffi::ACU_BOOL_IS_NULL, input, None) }
            pub fn is_not_null(input: &dyn Array) -> Result<BooleanArray, ArrowError> { boolean_op(ffi::ACU_BOOL_IS_NOT_NULL, input, None) }
        }

        /// `arrow::compute::kernels::bitwise` (arrow-arith/src/bitwise.rs): integer arrays only; the op at every slot,
        /// NullBuffer::union of the operands (array forms) or the left operand's nulls (scalar forms, not)
        pub mod bitwise {
            use super::*;
            fn bitwise_op<T: ArrowPrimitiveType>(op: i32, left: &PrimitiveArray<T>, right: Option<&PrimitiveArray<T>>,
                                                 scalar: Option<T::Native>) -> Result<PrimitiveArray<T>, ArrowError> {
                let dtype = native_code(&T::DATA_TYPE)
                    .ok_or_else(|| ArrowError::InvalidArgumentError(format!("Invalid bitwise operation: {}", T::DATA_TYPE)))?;
                let ctx = Context::current()?;
                let a = DeviceArray::upload(&ctx, left, false)?;
                let s = scalar.map(|v| PrimitiveArray::<T>::from_value(v, 1));
                let b = match (right, s.as_ref()) {
                    (Some(r), _) => Some(DeviceArray::upload(&ctx, r, false)?),
                    (None, Some(s)) => Some(DeviceArray::upload(&ctx, s, true)?),
                    (None, None) => None,
                };
                let mut out = ColumnOut::new(&ctx, &T::DATA_TYPE, left.len(), 0)?;
                ctx.check(unsafe { ffi::acu_bitwise(ctx.raw(), dtype, op, a.view(), b.as_ref().map_or(std::ptr::null(), |d| d.view() as *const _), out.array_out()) })?;
                Ok(out.finish(&T::DATA_TYPE)?.as_any().downcast_ref::<PrimitiveArray<T>>().unwrap().clone())
            }
            pub fn bitwise_and<T: ArrowPrimitiveType>(left: &PrimitiveArray<T>, right: &PrimitiveArray<T>) -> Result<PrimitiveArray<T>, ArrowError> { bitwise_op(ffi::ACU_BITWISE_AND, left, Some(right), None) }
            pub fn bitwise_or<T: ArrowPrimitiveType>(left: &PrimitiveArray<T>, right: &PrimitiveArray<T>) -> Result<PrimitiveArray<T>, ArrowError> { bitwise_op(ffi::ACU_BITWISE_OR, left, Some(right), None) }
            pub fn bitwise_xor<T: ArrowPrimitiveType>(left: &PrimitiveArray<T>, right: &PrimitiveArray<T>) -> Result<PrimitiveArray<T>, ArrowError> { bitwise_op(ffi::ACU_BITWISE_XOR, left, Some(right), None) }
            pub fn bitwise_and_not<T: ArrowPrimitiveType>(left: &PrimitiveArray<T>, right: &PrimitiveArray<T>) -> Result<PrimitiveArray<T>, ArrowError> { bitwise_op(ffi::ACU_BITWISE_AND_NOT, left, Some(right), None) }
            pub fn bitwise_shift_left<T: ArrowPrimitiveType>(left: &PrimitiveArray<T>, right: &PrimitiveArray<T>) -> Result<PrimitiveArray<T>, ArrowError> { bitwise_op(ffi::ACU_BITWISE_SHIFT_LEFT, left, Some(right), None) }
            pub fn bitwise_shift_right<T: ArrowPrimitiveType>(left: &PrimitiveArray<T>, right: &PrimitiveArray<T>) -> Result<PrimitiveArray<T>, ArrowError> { bitwise_op(ffi::ACU_BITWISE_SHIFT_RIGHT, left, Some(right), None) }
            pub fn bitwise_and_scalar<T: ArrowPrimitiveType>(array: &PrimitiveArray<T>, scalar: T::Native) -> Result<PrimitiveArray<T>, ArrowError> { bitwise_op(ffi::ACU_BITWISE_AND, array, None, Some(scalar)) }
            pub fn bitwise_or_scalar<T: ArrowPrimitiveType>(array: &PrimitiveArray<T>, scalar: T::Native) -> Result<PrimitiveArray<T>, ArrowError> { bitwise_op(ffi::ACU_BITWISE_OR, array, None, Some(scalar)) }
            pub fn bitwise_xor_scalar<T: ArrowPrimitiveType>(array: &PrimitiveArray<T>, scalar: T::Native) -> Result<PrimitiveArray<T>, ArrowError> { bitwise_op(ffi::ACU_BITWISE_XOR, array, None, Some(scalar)) }
            pub fn bitwise_shift_left_scalar<T: ArrowPrimitiveType>(array: &PrimitiveArray<T>, scalar: T::Native) -> Result<PrimitiveArray<T>, ArrowError> { bitwise_op(ffi::ACU_BITWISE_SHIFT_LEFT, array, None, Some(scalar)) }
            pub fn bitwise_shift_right_scalar<T: ArrowPrimitiveType>(array: &PrimitiveArray<T>, scalar: T::Native) -> Result<PrimitiveArray<T>, ArrowError> { bitwise_op(ffi::ACU_BITWISE_SHIFT_RIGHT, array, None, Some(scalar)) }
            pub fn bitwise_not<T: ArrowPrimitiveType>(array: &PrimitiveArray<T>) -> Result<PrimitiveArray<T>, ArrowError> { bitwise_op(ffi::ACU_BITWISE_NOT, array, None, None) }
        }
    }
}
