"""Invalid arguments to the C entries: the status and the bdf_last_error() text of every refusal, on a one-GPU context and on
multi-GPU contexts of every size the box has (a fleet of one GPU runs the whole fleet code path).  The entries are called
through ctypes, as the Rust shim calls them, so no check of the Python wrappers stands in front of them.  Where the two kinds
of context answer differently today, the table says so: each answer is pinned as it is."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

F64, I32, BOOL = 9, 2, 10
DATE32 = 1
INVALID, LENGTH_MISMATCH, UNSUPPORTED = 8, 1, 3
NULL_ARG = (INVALID, "null argument")
BAD_ARGS = (INVALID, "bad arguments")
BAD_VIEW = (INVALID, "bad view 0")
BAD_DTYPE = (INVALID, "invalid dtype 99")
MISMATCH = (LENGTH_MISMATCH, "Cannot perform math operation on arrays of different length")
SHARDED = (INVALID, "the columns are sharded differently over the GPUs (upload them in one bdf_upload_many call)")
ONE_GPU_COL = (INVALID, "a column of a one-GPU context was passed to a multi-GPU context")
NOT_A_DATE = (INVALID, "a column of dtype 9 does not hold this temporal type (dtype 2)")
SKIP = "skip"   # the call has no meaning on this kind of context


def _gpu_count():
    import torch

    return torch.cuda.device_count()


def _sizes():
    return [k for k in (1, 2, 3, 4, 8) if k <= _gpu_count()]


class Env:
    """One context under test, its device columns, and fresh host buffers for every call."""

    def __init__(self, rdf, ctx, other):
        from rust_dataframe_b200 import _native as N

        self.N, self.L, self.h = N, N.lib(), ctx.handle
        self.keep = []
        self.made = []
        self.A = self.upload([5, 3])      # A, B: the same chunk lengths
        self.B = self.upload([5, 3])
        self.C = self.upload([5, 4])      # chunk 1 differs
        self.D = self.upload([5])         # one chunk fewer, equal where it overlaps
        self.X = self.upload([5, 3], other.handle)   # a column of another (one-GPU) context
        self.agg = self.N.Agg4()

    def views(self, lens, np_dtype=np.float64, **over):
        v = (self.N.View * max(len(lens), 1))()
        for i, n in enumerate(lens):
            a = np.arange(max(n, 0), dtype=np_dtype)
            self.keep.append(a)
            v[i].values = a.ctypes.data if a.size else None
            v[i].len, v[i].offset, v[i].null_count = n, 0, 0
        for key, val in over.items():   # chunk0_offset=-1 -> v[0].offset = -1
            chunk, field = key.split("_", 1)
            setattr(v[int(chunk[5:])], field, val)
        return v

    def view_ptrs(self, *lens):
        return (C.POINTER(self.N.View) * len(lens))(*[C.cast(self.views(n), C.POINTER(self.N.View)) for n in lens])

    def outs(self, lens):
        o = (self.N.Out * max(len(lens), 1))()
        for i, n in enumerate(lens):
            a = np.zeros(max(n, 1), dtype=np.float64)
            m = np.zeros(max(n, 1), dtype=np.uint8)
            self.keep += [a, m]
            o[i].values, o[i].validity, o[i].len = a.ctypes.data, m.ctypes.data, n
        return o

    def upload(self, lens, handle=None):
        col = C.c_void_p()
        st = self.L.bdf_upload(handle or self.h, F64, len(lens), self.views(lens), 0, C.byref(col))
        assert st == 0, self.L.bdf_last_error()
        self.made.append((handle or self.h, col))
        return col

    def col_out(self):
        """Where an entry writes a result column; whatever it writes is freed after the case."""
        col = C.c_void_p()
        self.made.append((self.h, col))
        return C.byref(col)

    def cols(self, *cols):
        return (C.c_void_p * len(cols))(*[c.value for c in cols])

    def date32(self):
        t = self.N.TemporalTypeC(DATE32, 0, None)
        self.keep.append(t)
        return C.byref(t)

    def add_node(self):
        n = (self.N.ExprNode * 1)(self.N.ExprNode(0, 0, 1))
        self.keep.append(n)
        return n

    def close(self):
        for h, col in reversed(self.made):
            if col.value:
                self.L.bdf_col_free(h, col)


ADD, ABS, SUM = 0, 0, 0

# (name, call, answer on a one-GPU context, answer on a multi-GPU context or None for the same)
CASES = [
    # ---- host in / host out ----
    ("binary_bad_dtype", lambda e: e.L.bdf_binary(e.h, ADD, 99, 1, e.views([4]), 1, e.views([4]), e.outs([4])), BAD_DTYPE, None),
    ("binary_null_out", lambda e: e.L.bdf_binary(e.h, ADD, 99, 1, e.views([4]), 1, e.views([4]), None), BAD_DTYPE, BAD_ARGS),
    ("binary_negative_count", lambda e: e.L.bdf_binary(e.h, ADD, F64, -1, e.views([4]), 1, e.views([4]), e.outs([4])), BAD_ARGS, None),
    ("binary_null_left", lambda e: e.L.bdf_binary(e.h, ADD, F64, 1, None, 1, e.views([4]), e.outs([4])), BAD_ARGS, None),
    ("binary_length_mismatch", lambda e: e.L.bdf_binary(e.h, ADD, F64, 1, e.views([4]), 1, e.views([3]), e.outs([4])), MISMATCH, None),
    ("binary_bad_view", lambda e: e.L.bdf_binary(e.h, ADD, F64, 1, e.views([-1]), 1, e.views([-1]), e.outs([4])), BAD_VIEW, None),
    ("binary_bad_view_then_mismatch",
     lambda e: e.L.bdf_binary(e.h, ADD, F64, 2, e.views([4, 4], chunk0_offset=-1), 2, e.views([4, 3]), e.outs([4, 4])), MISMATCH, BAD_VIEW),
    ("unary_bad_dtype", lambda e: e.L.bdf_unary(e.h, ABS, 99, 1, e.views([4]), e.outs([4])), BAD_DTYPE, None),
    ("unary_negative_count", lambda e: e.L.bdf_unary(e.h, ABS, F64, -1, e.views([4]), e.outs([4])), BAD_ARGS, None),
    ("unary_null_in", lambda e: e.L.bdf_unary(e.h, ABS, F64, 1, None, e.outs([4])), BAD_ARGS, None),
    ("unary_bad_view", lambda e: e.L.bdf_unary(e.h, ABS, F64, 1, e.views([-1]), e.outs([4])), BAD_VIEW, None),
    ("unary_null_values", lambda e: e.L.bdf_unary(e.h, ABS, F64, 1, e.views([4], chunk0_values=None), e.outs([4])), BAD_VIEW, None),
    ("cast_bad_from_and_to", lambda e: e.L.bdf_cast(e.h, 98, 99, 1, e.views([4]), e.outs([4])),
     (INVALID, "invalid dtype 98"), BAD_DTYPE),
    ("cast_bad_to", lambda e: e.L.bdf_cast(e.h, F64, 99, 1, e.views([4]), e.outs([4])), BAD_DTYPE, None),
    ("cast_negative_count", lambda e: e.L.bdf_cast(e.h, F64, I32, -1, e.views([4]), e.outs([4])), BAD_ARGS, None),
    ("temporal_bad_fn", lambda e: e.L.bdf_temporal(e.h, 99, e.date32(), 0, 1, e.views([4], np.int32), e.outs([4])),
     (INVALID, "unknown temporal function 99"), None),
    ("temporal_null_type", lambda e: e.L.bdf_temporal(e.h, 0, None, 0, 1, e.views([4], np.int32), e.outs([4])),
     (INVALID, "null temporal type"), None),
    ("temporal_null_out", lambda e: e.L.bdf_temporal(e.h, 0, e.date32(), 0, 1, e.views([4], np.int32), None), BAD_ARGS, None),
    ("temporal_bad_view", lambda e: e.L.bdf_temporal(e.h, 0, e.date32(), 0, 1, e.views([-1], np.int32), e.outs([4])), BAD_VIEW, None),
    ("aggregate_null_is_some",
     lambda e: e.L.bdf_aggregate(e.h, SUM, 99, 1, e.views([4]), C.byref(C.c_double()), None), BAD_DTYPE, BAD_ARGS),
    ("aggregate_bad_dtype",
     lambda e: e.L.bdf_aggregate(e.h, SUM, 99, 1, e.views([4]), C.byref(C.c_double()), C.byref(C.c_int32())), BAD_DTYPE, None),
    ("aggregate_negative_count",
     lambda e: e.L.bdf_aggregate(e.h, SUM, F64, -1, e.views([4]), C.byref(C.c_double()), C.byref(C.c_int32())), BAD_ARGS, None),
    ("aggregate_bad_view",
     lambda e: e.L.bdf_aggregate(e.h, SUM, F64, 1, e.views([-1]), C.byref(C.c_double()), C.byref(C.c_int32())), BAD_VIEW, None),
    ("aggregate_bad_op",
     lambda e: e.L.bdf_aggregate(e.h, 99, F64, 1, e.views([4]), C.byref(C.c_double()), C.byref(C.c_int32())),
     (INVALID, "invalid aggregate op 99"), None),
    ("aggregate_all_null_out", lambda e: e.L.bdf_aggregate_all(e.h, 99, 1, e.views([4]), None), BAD_DTYPE, BAD_ARGS),
    ("aggregate_all_negative_count", lambda e: e.L.bdf_aggregate_all(e.h, F64, -1, e.views([4]), C.byref(e.agg)), BAD_ARGS, None),
    ("aggregate_all_bad_view", lambda e: e.L.bdf_aggregate_all(e.h, F64, 1, e.views([-1]), C.byref(e.agg)), BAD_VIEW, None),
    ("avg_null_is_some", lambda e: e.L.bdf_avg(e.h, 99, 1, e.views([4]), C.byref(C.c_double()), None), BAD_DTYPE, BAD_ARGS),
    ("avg_bad_view", lambda e: e.L.bdf_avg(e.h, F64, 1, e.views([-1]), C.byref(C.c_double()), C.byref(C.c_int32())), BAD_VIEW, None),
    ("moments_bool", lambda e: e.L.bdf_moments(e.h, BOOL, 1, e.views([4]), C.byref(e.N.MomentRec())),
     (UNSUPPORTED, "the statistics need a numeric column"), None),
    ("moments_bad_dtype", lambda e: e.L.bdf_moments(e.h, 99, 1, e.views([4]), C.byref(e.N.MomentRec())), BAD_DTYPE, None),
    ("moments_null_out", lambda e: e.L.bdf_moments(e.h, F64, 1, e.views([4]), None), BAD_ARGS, None),
    ("moments_bad_view", lambda e: e.L.bdf_moments(e.h, F64, 1, e.views([-1]), C.byref(e.N.MomentRec())), BAD_VIEW, None),
    ("distinct_null_out", lambda e: e.L.bdf_distinct(e.h, F64, 1, e.views([4]), None), BAD_ARGS,
     (UNSUPPORTED, "distinct values need every row of the column on one GPU (as sort / group-by / join): use a one-GPU context")),
    # ---- uploads and generated columns ----
    ("upload_bad_dtype", lambda e: e.L.bdf_upload(e.h, 99, 1, e.views([4]), 0, e.col_out()), BAD_DTYPE, None),
    ("upload_null_out", lambda e: e.L.bdf_upload(e.h, F64, 1, e.views([4]), 0, None), BAD_ARGS, None),
    ("upload_negative_count", lambda e: e.L.bdf_upload(e.h, F64, -1, e.views([4]), 0, e.col_out()), BAD_ARGS, None),
    ("upload_bad_view", lambda e: e.L.bdf_upload(e.h, F64, 1, e.views([-1]), 0, e.col_out()), BAD_VIEW, None),
    ("upload_many_negative_count",
     lambda e: e.L.bdf_upload_many(e.h, -1, (C.c_int32 * 1)(F64), (C.c_int64 * 1)(1), None, 0, None), BAD_ARGS, None),
    ("upload_many_bad_column",
     lambda e: e.L.bdf_upload_many(e.h, 2, (C.c_int32 * 2)(F64, F64), (C.c_int64 * 2)(1, -1),
                                   e.view_ptrs([4], [4]), 0, (C.c_void_p * 2)()),
     (INVALID, "bad arguments for column 1"), None),
    ("upload_many_bad_dtype",
     lambda e: e.L.bdf_upload_many(e.h, 2, (C.c_int32 * 2)(F64, 99), (C.c_int64 * 2)(1, 1),
                                   e.view_ptrs([4], [4]), 0, (C.c_void_p * 2)()), BAD_DTYPE, None),
    ("generate_bad_kind", lambda e: e.L.bdf_generate(e.h, F64, 7, 0.0, 1.0, 1, 0, 1, (C.c_int64 * 1)(4), 0, 0, e.col_out()), BAD_ARGS, None),
    ("generate_bad_dtype", lambda e: e.L.bdf_generate(e.h, 99, 0, 0.0, 1.0, 1, 0, 1, (C.c_int64 * 1)(4), 0, 0, e.col_out()), BAD_DTYPE, None),
    ("generate_negative_chunk",
     lambda e: e.L.bdf_generate(e.h, F64, 0, 0.0, 1.0, 1, 0, 2, (C.c_int64 * 2)(4, -1), 0, 0, e.col_out()),
     (INVALID, "negative chunk length"), None),
    # ---- device columns ----
    ("binary_dev_null_out", lambda e: e.L.bdf_binary_dev(e.h, ADD, e.A, e.B, None), NULL_ARG, None),
    ("binary_dev_length_mismatch", lambda e: e.L.bdf_binary_dev(e.h, ADD, e.A, e.C, e.col_out()), MISMATCH, None),
    ("binary_dev_chunk_counts", lambda e: e.L.bdf_binary_dev(e.h, ADD, e.A, e.D, e.col_out()),
     (0, ""), (UNSUPPORTED, "columns with different numbers of chunks on a multi-GPU context")),
    ("binary_dev_one_gpu_column", lambda e: e.L.bdf_binary_dev(e.h, ADD, e.A, e.X, e.col_out()), SKIP, ONE_GPU_COL),
    ("binary_dev_bad_op", lambda e: e.L.bdf_binary_dev(e.h, 99, e.A, e.B, e.col_out()), (INVALID, "invalid binary op 99"), None),
    ("unary_dev_null_in", lambda e: e.L.bdf_unary_dev(e.h, ABS, None, e.col_out()), NULL_ARG, None),
    ("cast_dev_null_out", lambda e: e.L.bdf_cast_dev(e.h, I32, e.A, None), NULL_ARG, None),
    ("cast_dev_bad_to", lambda e: e.L.bdf_cast_dev(e.h, 99, e.A, e.col_out()), BAD_DTYPE, None),
    ("temporal_dev_bad_fn", lambda e: e.L.bdf_temporal_dev(e.h, 99, e.date32(), 0, None, None),
     (INVALID, "unknown temporal function 99"), None),
    ("temporal_dev_not_a_date", lambda e: e.L.bdf_temporal_dev(e.h, 0, e.date32(), 0, e.A, e.col_out()), NOT_A_DATE, None),
    ("temporal_dev_null_out", lambda e: e.L.bdf_temporal_dev(e.h, 0, e.date32(), 0, e.A, None), NULL_ARG, None),
    ("temporal_binary_dev_null_type",
     lambda e: e.L.bdf_temporal_binary_dev(e.h, 9, None, e.A, e.date32(), e.B, e.col_out()),
     (INVALID, "unknown two-column temporal function 9"), NULL_ARG),
    ("temporal_binary_dev_null_column", lambda e: e.L.bdf_temporal_binary_dev(e.h, 0, e.date32(), None, e.date32(), e.B, e.col_out()),
     NULL_ARG, None),
    ("temporal_binary_dev_not_a_date", lambda e: e.L.bdf_temporal_binary_dev(e.h, 0, e.date32(), e.A, e.date32(), e.B, e.col_out()),
     NOT_A_DATE, None),
    ("aggregate_dev_null_is_some", lambda e: e.L.bdf_aggregate_dev(e.h, SUM, e.A, C.byref(C.c_double()), None), NULL_ARG, None),
    ("aggregate_dev_bad_op", lambda e: e.L.bdf_aggregate_dev(e.h, 99, e.A, C.byref(C.c_double()), C.byref(C.c_int32())),
     (INVALID, "invalid aggregate op 99"), None),
    ("aggregate_all_dev_null_out", lambda e: e.L.bdf_aggregate_all_dev(e.h, e.A, None), NULL_ARG, None),
    ("aggregate_all_dev_one_gpu_column", lambda e: e.L.bdf_aggregate_all_dev(e.h, e.X, C.byref(e.agg)), SKIP, ONE_GPU_COL),
    ("avg_dev_null_out", lambda e: e.L.bdf_avg_dev(e.h, e.A, None, C.byref(C.c_int32())), NULL_ARG, None),
    ("moments_dev_null_out", lambda e: e.L.bdf_moments_dev(e.h, e.A, None), NULL_ARG, None),
    ("binary_agg_dev_null_agg", lambda e: e.L.bdf_binary_agg_dev(e.h, ADD, e.A, e.B, e.col_out(), None), NULL_ARG, None),
    ("binary_agg_dev_length_mismatch", lambda e: e.L.bdf_binary_agg_dev(e.h, ADD, e.A, e.C, e.col_out(), C.byref(e.agg)), MISMATCH, None),
    ("binary_agg_dev_chunk_counts", lambda e: e.L.bdf_binary_agg_dev(e.h, ADD, e.A, e.D, e.col_out(), C.byref(e.agg)), (0, ""), SHARDED),
    ("binary_agg_dev_async_null_fut", lambda e: e.L.bdf_binary_agg_dev_async(e.h, ADD, e.A, e.B, e.col_out(), None), NULL_ARG, None),
    ("eval_expr_dev_null_nodes", lambda e: e.L.bdf_eval_expr_dev(e.h, 2, e.cols(e.A, e.B), 1, None, e.col_out()), NULL_ARG, BAD_ARGS),
    ("eval_expr_dev_chunk_counts", lambda e: e.L.bdf_eval_expr_dev(e.h, 2, e.cols(e.A, e.D), 1, e.add_node(), e.col_out()), (0, ""), SHARDED),
    ("eval_expr_dev_length_mismatch", lambda e: e.L.bdf_eval_expr_dev(e.h, 2, e.cols(e.A, e.C), 1, e.add_node(), e.col_out()),
     MISMATCH, SHARDED),
    ("eval_expr_dev_one_gpu_column", lambda e: e.L.bdf_eval_expr_dev(e.h, 2, e.cols(e.A, e.X), 1, e.add_node(), e.col_out()),
     SKIP, (INVALID, "null input column")),
    ("eval_expr_agg_dev_null_agg", lambda e: e.L.bdf_eval_expr_agg_dev(e.h, 2, e.cols(e.A, e.B), 1, e.add_node(), e.col_out(), None),
     NULL_ARG, None),
    ("eval_expr_agg_dev_null_inputs", lambda e: e.L.bdf_eval_expr_agg_dev(e.h, 2, None, 1, e.add_node(), e.col_out(), C.byref(e.agg)),
     NULL_ARG, BAD_ARGS),
    ("eval_expr_agg_dev_chunk_counts",
     lambda e: e.L.bdf_eval_expr_agg_dev(e.h, 2, e.cols(e.A, e.D), 1, e.add_node(), e.col_out(), C.byref(e.agg)), (0, ""), SHARDED),
    ("eval_expr_agg_dev_async_null_fut",
     lambda e: e.L.bdf_eval_expr_agg_dev_async(e.h, 2, e.cols(e.A, e.B), 1, e.add_node(), e.col_out(), None), NULL_ARG, BAD_ARGS),
    ("download_null_out", lambda e: e.L.bdf_download(e.h, e.A, None), NULL_ARG, None),
    ("download_begin_null_out", lambda e: e.L.bdf_download_begin(e.h, e.A, None), NULL_ARG, None),
    ("download_end_null_out", lambda e: e.L.bdf_download_end(e.h, e.A, None), NULL_ARG, None),
    ("download_capacity", lambda e: e.L.bdf_download(e.h, e.A, e.outs([4, 3])),
     (INVALID, "output chunk 0 has capacity 4, result has 5 rows"), None),
    ("download_one_gpu_column", lambda e: e.L.bdf_download(e.h, e.X, e.outs([5, 3])), SKIP, NULL_ARG),
]

# A null context: the entries that check their arguments before the context answer for them first.
NULL_CTX = (INVALID, "null context")
NULL_CTX_CASES = [
    ("binary", lambda L, N: L.bdf_binary(None, ADD, 99, 1, None, 1, None, None), NULL_CTX),
    ("unary", lambda L, N: L.bdf_unary(None, ABS, 99, -1, None, None), NULL_CTX),
    ("cast", lambda L, N: L.bdf_cast(None, 98, 99, -1, None, None), NULL_CTX),
    ("temporal", lambda L, N: L.bdf_temporal(None, 99, None, 0, -1, None, None), NULL_CTX),
    ("aggregate", lambda L, N: L.bdf_aggregate(None, SUM, 99, -1, None, None, None), NULL_CTX),
    ("aggregate_all", lambda L, N: L.bdf_aggregate_all(None, 99, -1, None, None), NULL_CTX),
    ("avg", lambda L, N: L.bdf_avg(None, 99, -1, None, None, None), NULL_CTX),
    ("moments", lambda L, N: L.bdf_moments(None, BOOL, -1, None, None), NULL_CTX),
    ("distinct", lambda L, N: L.bdf_distinct(None, BOOL, -1, None, None), NULL_CTX),
    ("upload", lambda L, N: L.bdf_upload(None, 99, -1, None, 0, None), NULL_CTX),
    ("upload_many", lambda L, N: L.bdf_upload_many(None, -1, None, None, None, 0, None), NULL_CTX),
    ("generate", lambda L, N: L.bdf_generate(None, 99, 7, 0.0, 1.0, 1, 0, -1, None, 0, 0, None), NULL_CTX),
    ("binary_dev", lambda L, N: L.bdf_binary_dev(None, ADD, None, None, None), NULL_CTX),
    ("unary_dev", lambda L, N: L.bdf_unary_dev(None, ABS, None, None), NULL_CTX),
    ("cast_dev", lambda L, N: L.bdf_cast_dev(None, 99, None, None), NULL_CTX),
    ("temporal_dev", lambda L, N: L.bdf_temporal_dev(None, 99, None, 0, None, None), (INVALID, "null temporal type")),
    ("temporal_binary_dev", lambda L, N: L.bdf_temporal_binary_dev(None, 9, None, None, None, None, None), NULL_CTX),
    ("aggregate_dev", lambda L, N: L.bdf_aggregate_dev(None, 99, None, None, None), NULL_CTX),
    ("aggregate_all_dev", lambda L, N: L.bdf_aggregate_all_dev(None, None, None), NULL_CTX),
    ("avg_dev", lambda L, N: L.bdf_avg_dev(None, None, None, None), NULL_CTX),
    ("moments_dev", lambda L, N: L.bdf_moments_dev(None, None, None), NULL_CTX),
    ("binary_agg_dev", lambda L, N: L.bdf_binary_agg_dev(None, ADD, None, None, None, None), NULL_CTX),
    ("binary_agg_dev_async", lambda L, N: L.bdf_binary_agg_dev_async(None, ADD, None, None, None, None), NULL_CTX),
    ("eval_expr_dev", lambda L, N: L.bdf_eval_expr_dev(None, 0, None, 0, None, None), NULL_CTX),
    ("eval_expr_agg_dev", lambda L, N: L.bdf_eval_expr_agg_dev(None, 0, None, 0, None, None, None), NULL_CTX),
    ("eval_expr_agg_dev_async", lambda L, N: L.bdf_eval_expr_agg_dev_async(None, 0, None, 0, None, None, None), NULL_CTX),
    ("download", lambda L, N: L.bdf_download(None, None, None), NULL_CTX),
    ("download_begin", lambda L, N: L.bdf_download_begin(None, None, None), NULL_CTX),
    ("download_end", lambda L, N: L.bdf_download_end(None, None, None), NULL_CTX),
]


@pytest.fixture(scope="module")
def other(rdf):
    if not _gpu_count():
        pytest.skip("no GPU")
    ctx = rdf.Context(0)
    yield ctx
    ctx.close()


@pytest.fixture(scope="module", params=["one"] + [f"fleet{k}" for k in _sizes()])
def env(request, rdf, other):
    ctx = rdf.Context(0) if request.param == "one" else rdf.Context.multi(int(request.param[5:]))
    e = Env(rdf, ctx, other)
    e.fleet = request.param != "one"
    yield e
    e.close()
    ctx.close()


def test_every_refusal_keeps_its_status_and_message(env):
    got, want = {}, {}
    for name, call, one, fleet in CASES:
        expect = fleet if (env.fleet and fleet is not None) else one
        if expect == SKIP:
            continue
        st = call(env)
        msg = (env.L.bdf_last_error() or b"").decode() if st else ""
        got[name], want[name] = (st, msg), tuple(expect)
        for h, col in env.made[5:]:   # results of the calls that succeed on one kind of context
            if col.value:
                env.L.bdf_col_free(h, col)
                col.value = None
        env.keep.clear()
    assert {k: v for k, v in got.items() if v != want[k]} == {k: v for k, v in want.items() if v != got[k]}


def test_a_null_context_answers_first(rdf):
    from rust_dataframe_b200 import _native as N

    L = N.lib()
    got = {name: (st := call(L, N), (L.bdf_last_error() or b"").decode() if st else "") for name, call, _ in NULL_CTX_CASES}
    assert got == {name: want for name, _, want in NULL_CTX_CASES}
