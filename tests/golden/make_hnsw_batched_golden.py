"""Regenerates tests/golden/hnsw_batched_graphs.json: the SHA-256 of get_trained_state() after seeded
b200vs_hnsw_add_batched builds with batches larger than one (DESIGN §4.4).  Such a graph has no second builder to be
compared with, so these hashes pin it: a change of the construction search, the link rule or the tie-break shows up as a
different hash.  Needs a GPU:
    python tests/golden/make_hnsw_batched_golden.py          # rewrites the file
The cases cover both forms of the construction search: the merged array (default batch, no tombstones) and the two heaps
(tombstones from a delete and an upsert between calls, with L2 and with cosine; efc above the merged array's limit).
The stored hashes were recorded on an H100 with the library of commit ce3b82d, the last one whose construction search was
its own copy of the search walk; the shared walk must rebuild the same graphs."""
import hashlib
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))),
                                "dingo-store_b200", "python"))
import b200vs  # noqa: E402
from b200vs import COSINE, HNSW, IP, L2  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hnsw_batched_graphs.json")

# name -> (metric, n, d, M, efc, batch, calls, tombstones between calls)
CASES = {
    "l2_default_batch": (L2, 6000, 32, 16, 100, 0, 2, False),
    "ip_default_batch": (IP, 6000, 32, 16, 100, 0, 2, False),
    "cosine_default_batch": (COSINE, 6000, 32, 16, 100, 0, 2, False),
    "l2_delete_upsert_heap_form": (L2, 6000, 32, 12, 80, 0, 2, True),
    "cosine_delete_upsert_heap_form": (COSINE, 6000, 32, 12, 80, 0, 2, True),
    "l2_efc1100_heap_form": (L2, 3000, 8, 6, 1100, 0, 2, False),
    "cosine_batch257": (COSINE, 6000, 32, 16, 100, 257, 2, False),
}


def graph_hash(name):
    metric, n, d, M, efc, batch, calls, tombstones = CASES[name]
    rng = np.random.default_rng(n + d + M + efc + batch)
    xb = rng.random((n, d)).astype(np.float32)
    labels = np.arange(1000, 1000 + n, dtype=np.int64)
    ix = b200vs.Index(HNSW, metric, d, hnsw_m=M, hnsw_efc=efc, max_elements=4 * n)
    step = (n + calls - 1) // calls
    for a in range(0, n, step):
        if tombstones and a > 0:
            ix.delete(labels[:a:7])
            ups = labels[3:a:11]  # some of them deleted just above
            ix.add_batched(rng.random((len(ups), d)).astype(np.float32), ups, batch=batch)
        ix.add_batched(xb[a:a + step], labels[a:a + step], batch=batch)
    return hashlib.sha256(np.ascontiguousarray(ix.get_trained_state()).tobytes()).hexdigest()


def main():
    out = {name: graph_hash(name) for name in CASES}
    with open(OUT, "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
