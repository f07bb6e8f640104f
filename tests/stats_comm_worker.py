"""One rank of the two-rank statistics run (tests/test_stats_gpu.py): argv = unique id (hex), rank, world.  Every rank builds the
same column from a fixed seed, keeps chunks i with i mod world == rank, attaches to the communicator and prints the merged moment
record of the whole column, which must be the same bits on every rank."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    import rust_dataframe_b200 as rdf
    import stats_oracle as so

    uid, rank, world = bytes.fromhex(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3])
    rng = np.random.default_rng(20261015)
    lens = [100_000, 1, 0, 70_001, 333]
    chunks = [rdf.PrimitiveArray.from_numpy(1e6 + rng.uniform(-1, 1, n), rng.random(n) >= 0.1) for n in lens]
    ctx = rdf.Context(rank)
    ctx.comm_attach(uid, rank, world)
    mine = [c for i, c in enumerate(chunks) if i % world == rank]
    rec = rdf.AggregateFunctions.moments(mine, ctx=ctx)
    err = so.within_bars(rec, so.exact_moments(so.valid_values(chunks)))
    if err:
        print("bars failed:", err, file=sys.stderr)
        sys.exit(1)
    ctx.comm_detach()
    ctx.close()
    print(json.dumps({k: float(v).hex() if k != "count" else v for k, v in rec.items()}))


if __name__ == "__main__":
    main()
