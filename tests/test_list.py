"""CPU checks of the list functions: the oracle against the reference's six array tests, against pyarrow and against
independent per-list Python; the host ListArray; the IPC reader's description of List<T> columns (no context, no GPU)."""
import json
import math
import os

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import list_oracle as lo

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "array_functions.json")))
NUMERIC = [pa.int8(), pa.int16(), pa.int32(), pa.int64(), pa.uint8(), pa.uint16(), pa.uint32(), pa.uint64(), pa.float32(), pa.float64()]


def golden_lists(cast=int):
    v, o = GOLDEN["values"], GOLDEN["offsets"]
    return [[cast(x) for x in v[o[i]:o[i + 1]]] for i in range(len(o) - 1)]


def flat_offsets(lists):
    off, vals = [0], []
    for l in lists:
        vals.extend(l or [])
        off.append(len(vals))
    return off, vals


@pytest.mark.parametrize("cast", [int, float])
def test_oracle_reproduces_the_reference_contains_tests(cast):
    g = GOLDEN["contains"]
    assert [lo.array_contains(l, cast(g["value"])) for l in golden_lists(cast)] == g["expected"]


def test_oracle_reproduces_the_reference_position_remove_sort_tests():
    lists = golden_lists()
    assert [lo.array_position(l, 2) for l in lists] == GOLDEN["position"]["expected"]
    off, vals = flat_offsets([lo.array_remove(l, 2) for l in lists])
    assert off[:-1] == GOLDEN["remove"]["offsets"] and len(vals) == GOLDEN["remove"]["values_len"]
    off, vals = flat_offsets([lo.array_sort(l) for l in lists])
    assert off[:-1] == GOLDEN["sort"]["offsets"] and vals == GOLDEN["sort"]["values"]


def random_lists(rng, n, float_values=False):
    out = []
    pool = [0.0, -0.0, float("nan"), 1.5, -2.0, 3.0] if float_values else [0, 1, 2, 3, -4]
    for _ in range(n):
        r = rng.random()
        if r < 0.1:
            out.append(None)
        elif r < 0.2:
            out.append([])
        else:
            out.append([None if rng.random() < 0.15 else pool[rng.integers(len(pool))] for _ in range(rng.integers(1, 9))])
    return out


@pytest.mark.parametrize("seed", [1, 2])
def test_size_and_explode_against_pyarrow(seed):
    rng = np.random.default_rng(seed)
    lists = random_lists(rng, 300)
    arr = pa.array(lists, pa.list_(pa.int64()))
    want_size = [-1 if x is None else x for x in pc.list_value_length(arr).to_pylist()]
    assert [lo.size(l) for l in lists] == want_size
    rows, values = lo.explode(lists)
    assert values == pc.list_flatten(arr).to_pylist()
    assert rows == pc.list_parent_indices(arr).to_pylist()


def _bits(x):
    if x is None:
        return None
    if isinstance(x, float):
        return ("f", np.float64(x).view(np.uint64).item()) if not math.isnan(x) else ("nan",)
    return ("i", int(x))


@pytest.mark.parametrize("float_values", [False, True])
def test_oracle_against_independent_python(float_values):
    rng = np.random.default_rng(5)
    A, B = random_lists(rng, 400, float_values), random_lists(rng, 400, float_values)

    def norm(x):   # a value of the key space: NaN one value, -0.0 == 0.0, None one value
        if x is None:
            return "null"
        if isinstance(x, float) and math.isnan(x):
            return "nan"
        return x + 0.0 if isinstance(x, float) else x

    def dict_distinct(xs):   # dict keys keep first-insertion order
        d = {}
        for x in xs:
            d.setdefault(norm(x), x)
        return list(d.values())

    v = 0.0 if float_values else 2
    for a, b in zip(A, B):
        if a is None:
            assert lo.array_sort(a) == [] and lo.array_distinct(a) == [] and lo.array_union(a, b) == []
            continue
        assert [_bits(x) for x in lo.array_distinct(a)] == [_bits(x) for x in dict_distinct(a)]
        assert [_bits(x) for x in lo.array_union(a, b)] == [_bits(x) for x in dict_distinct(a + (b or []))]
        bset = {norm(x) for x in (b or [])}
        assert [_bits(x) for x in lo.array_except(a, b)] == [_bits(x) for x in dict_distinct(a) if norm(x) not in bset]
        assert [_bits(x) for x in lo.array_intersect(a, b)] == [_bits(x) for x in dict_distinct(a) if norm(x) in bset]
        s = lo.array_sort(a)
        nn = [x for x in a if x is not None]
        nums = sorted([x for x in nn if not (isinstance(x, float) and math.isnan(x))])
        nans = [x for x in nn if isinstance(x, float) and math.isnan(x)]
        assert [_bits(x) for x in s] == [_bits(x) for x in nums + nans + [None] * (len(a) - len(nn))]
        assert [_bits(x) for x in lo.array_remove(a, v)] == [_bits(x) for x in a if x is None or norm(x) != norm(v)]
        assert lo.array_position(a, v) == next((i + 1 for i, x in enumerate(a) if x is not None and norm(x) == norm(v)), 0)
        assert lo.array_repeat(a, 3) == a * 3
        if a:
            valid = [x for x in a if x is not None]
            if valid and not float_values:
                assert lo.array_max(a) == max(valid) and lo.array_min(a) == min(valid)
        else:
            with pytest.raises(lo.Panic):
                lo.array_max(a)


def test_float_min_max_follow_total_order():
    assert math.copysign(1.0, lo.array_min([0.0, -0.0])) < 0 and math.copysign(1.0, lo.array_max([-0.0, 0.0])) > 0
    assert math.isnan(lo.array_max([1.0, float("nan")])) and lo.array_min([1.0, float("nan")]) == 1.0
    assert lo.array_max([None, None]) is None and lo.array_max(None) is None


def test_host_list_array_round_trips(rdf):
    items = [[1, 2], None, [], [None, 3]]
    a = rdf.ListArray.from_pylist(rdf.I16, items)
    assert a.to_pylist() == items
    arr = pa.array([[5], [1, None], None, [7, 8, 9]], pa.list_(pa.int32())).slice(1)
    b = rdf.ListArray.from_arrow(arr)
    assert b.offset == 1 and b.to_pylist() == arr.to_pylist()


def test_ipc_describes_list_columns_without_a_gpu(rdf, tmp_path):
    cols, names = [], []
    for t in NUMERIC:
        names.append(f"l_{t}")
        cols.append(pa.array([[1, 2], None, [], [3]], pa.list_(t)))
    extra = {"large": pa.array([[1]] * 4, pa.large_list(pa.int32())), "nested": pa.array([[[1]]] * 4, pa.list_(pa.list_(pa.int32()))),
             "bools": pa.array([[True]] * 4, pa.list_(pa.bool_())), "plain": pa.array([1, 2, 3, 4], pa.int32())}
    for k, v in extra.items():
        names.append(k)
        cols.append(v)
    path = str(tmp_path / "lists.arrow")
    table = pa.table(cols, names=names)
    with pa.OSFile(path, "wb") as sink, pa.ipc.new_file(sink, table.schema) as w:
        w.write_table(table)
    with rdf.IpcFile(path) as f:
        for i, t in enumerate(NUMERIC):
            assert f.schema[i][1] == -1                      # the column path is unchanged
            assert f.list_columns[f"l_{t}"] == rdf.native.LIST_BASE + i
        for k in ("large", "nested", "bools", "plain"):
            assert k not in f.list_columns
        assert dict((n, d) for n, d, _ in f.schema)["plain"] == rdf.I32


def test_header_declares_the_list_abi(rdf):
    text = open(os.path.join(os.path.dirname(HERE), "include", "b200df.h")).read()
    assert "#define BDF_ABI_VERSION 3" in text and "#define BDF_LIST_BASE 32" in text
    N = rdf.native
    assert N.KERNEL_NAMES[N.K_LIST] == "list"
    import ctypes as C
    assert C.sizeof(N.ListView) == 40 + C.sizeof(N.View) and C.sizeof(N.ListOut) == 56
