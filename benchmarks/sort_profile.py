#!/usr/bin/env python
"""One 1e8-row Float64 sort (k_sort_keys, 8 x [k_radix_hist, k_scan_one, k_radix_scatter]) and one take, for ncu:
   ncu --set full -k regex:"k_sort_keys|k_radix_hist|k_radix_scatter|k_take" --launch-skip 15 -c 3 python benchmarks/sort_profile.py"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import rust_dataframe_b200 as rdf  # noqa: E402

ctx = rdf.default_context()
lens = [4_000_000] * 25
a = rdf.Column.generate(rdf.F64, lens, 0, -1e3, 1e3, col_id=0)
idx = rdf.sort_indices([(a, False)])
t = a.take(idx)
ctx.synchronize()
print("sorted", t.count())
