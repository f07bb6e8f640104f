"""Writes array_functions.json: the fixed data and every asserted result of the reference's six array tests
(src/functions/array.rs, mod tests: test_array_contains_i32s / _i64s / _f64s, test_array_position, test_array_remove,
test_array_sort).  The numbers are copied from those tests' literals; nothing here is computed."""
import json
import os

VALUES = [0, 0, 0, 1, 2, 1, 3, 4, 5, 1, 3, 2, 3, 2, 8, 3]   # every test's value array (Int32, Int64 or Float64)
OFFSETS = [0, 3, 6, 8, 12, 14, 16]

GOLDEN = {
    "values": VALUES,
    "offsets": OFFSETS,
    "contains": {"types": ["Int32", "Int64", "Float64"], "value": 2, "expected": [False, True, False, True, True, False]},
    "position": {"type": "Int64", "value": 2, "expected": [0, 2, 0, 4, 2, 0]},
    "remove": {"type": "Int64", "value": 2, "len": 6, "values_len": 13, "offsets": [0, 3, 5, 7, 10, 11]},
    "sort": {"type": "Int64", "len": 6, "values_len": 16, "offsets": [0, 3, 6, 8, 12, 14],
             "values": [0, 0, 0, 1, 1, 2, 3, 4, 1, 2, 3, 5, 2, 3, 3, 8]},
}

if __name__ == "__main__":
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "array_functions.json"), "w") as f:
        json.dump(GOLDEN, f, indent=1)
        f.write("\n")
