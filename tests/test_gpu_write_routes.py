"""Every write entry point of every index type, on small seeded indexes (one GPU).

One index kind at a time, the same rows are written by every route the type has: the host add in one call and in two, the
device add without and with the caller's lists, the sharded add and device add at a world of one, the batched HNSW build
alone and through the shard, b200vs_save then b200vs_load into a fresh index, the shard's save then load at a world of
one, and b200vs_rebuild_from.  Routes that must build the same index must give byte-equal export_lists (offsets, ids, and
rows or codes) and bit-equal search results; the loaded and restored rows of a cosine index are the saved rows, bit for
bit, so nothing is normalised twice.  An upsert of a subset must equal adding the other rows and then the subset.  Every
refused (kind, write entry point) pair must return the recorded status code and b200vs_last_error text, and a refused
collective add must leave the index as it was."""
import numpy as np
import pytest

import b200vs
from b200vs import BINARY_FLAT, BINARY_IVF_FLAT, COSINE, FLAT, HAMMING, HNSW, IP, IVF_FLAT, IVF_PQ, L2
from gpu_util import require_gpu

pytestmark = pytest.mark.gpu
D, BITS, NLIST, NPROBE, K, N, PQ_M = 32, 256, 16, 6, 10, 2000, 8


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def _rows(n, seed, d=D):
    return np.random.default_rng(seed).standard_normal((n, d)).astype(np.float32)


def _bits(n, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, BITS // 8), dtype=np.uint8)


class Kind:
    """How to make a fresh index of one kind, its rows, and how to read it back."""

    def __init__(self, name):
        self.name = name
        self.binary = name.startswith("binary")
        self.hnsw = name.startswith("hnsw")
        self.pq = name.startswith(("ivf_pq8", "ivf_pq4"))
        self.pqflat = name.startswith("ivf_pqflat")
        self.ivf = name.startswith(("ivf_flat", "binary_ivf")) or self.pq
        self.rows_sharded = name.startswith(("flat", "hnsw", "binary_flat"))
        self.nbits = 4 if name.startswith("ivf_pq4") else 8
        self.metric = HAMMING if self.binary else {"l2": L2, "ip": IP, "cos": COSINE}[name.split("_")[-1]]
        self.x = _bits(N, 1) if self.binary else _rows(N, 1)
        self.q = _bits(64, 2) if self.binary else _rows(64, 2)
        self.ids = np.arange(1, N + 1, dtype=np.int64)
        self.blob = None
        if self.ivf:  # every trained index of the kind shares one trained state
            ix = self.new(trained=False)
            ix.train(_rows(max(256 * NLIST, 256 << self.nbits) + 1000, 3) if self.pq else self.x)
            self.blob = ix.get_trained_state()

    def new(self, trained=True, max_elements=2 * N):
        if self.binary:
            ix = b200vs.Index(BINARY_FLAT if self.name == "binary_flat" else BINARY_IVF_FLAT, HAMMING, BITS, nlist=NLIST)
        elif self.name.startswith("flat"):
            ix = b200vs.Index(FLAT, self.metric, D)
        elif self.name.startswith("ivf_flat"):
            ix = b200vs.Index(IVF_FLAT, self.metric, D, nlist=NLIST)
        elif self.hnsw:
            ix = b200vs.Index(HNSW, self.metric, D, hnsw_m=16, hnsw_efc=100, max_elements=max_elements)
        else:
            ix = b200vs.Index(IVF_PQ, self.metric, D, nlist=NLIST, pq_m=PQ_M, pq_nbits=self.nbits)
        if trained and self.blob is not None:
            ix.set_trained_state(self.blob)
        elif trained and self.pqflat:
            ix.train(_rows(100, 3))  # too few rows for IVF-PQ: the inner Flat index
        return ix

    def shard(self, ix):
        return (b200vs.BinaryShard if self.binary else b200vs.Shard)(ix, 0, 1, None)

    def read(self, ix):
        """(export_lists, top-k search) of ix."""
        nl = NLIST if self.ivf else 1
        if self.pq:
            exp = ix.export_lists(nl, with_vectors=False, code_size=(PQ_M * self.nbits + 7) // 8)
        else:
            exp = ix.export_lists(nl)
        return [a for a in exp if a is not None] + list(ix.search(self.q, K, nprobe=NPROBE))


def _same(a, b):
    return len(a) == len(b) and all(
        np.asarray(x).shape == np.asarray(y).shape and np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))
        for x, y in zip(a, b))


def _refusal(call):
    try:
        call()
    except b200vs.B200VSError as e:
        return [e.code, e.msg]
    return "ok"


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def observe(kind_name, tmp_path):
    """{route: "same" | "differs" | "ok" | [status, last_error]} of one index kind."""
    import torch

    k = Kind(kind_name)
    x, ids, n = k.x, k.ids, N
    obs = {}

    ref = k.new()
    ref.add(x, ids)
    want = k.read(ref)

    def compare(route, build):
        """build(ix) writes the rows into the fresh, trained index ix; a refusal is recorded as such."""
        ix = k.new()
        got = _refusal(lambda: build(ix))
        obs[route] = got if got != "ok" else ("same" if _same(k.read(ix), want) else "differs")
        return ix

    def add_2(ix):
        ix.add(x[: n // 3], ids[: n // 3])
        ix.add(x[n // 3:], ids[n // 3:])

    compare("add_2", add_2)

    xd, idd = _dev(x), _dev(ids)
    compare("add_device", lambda ix: ix.add_device(n, xd.data_ptr(), idd.data_ptr()))
    if k.ivf and not k.binary:
        lists = torch.empty(n, dtype=torch.int64, device="cuda")
        ref.assign_device(n, xd.data_ptr(), lists.data_ptr())
        compare("add_device_lists", lambda ix: ix.add_device(n, xd.data_ptr(), idd.data_ptr(), lists.data_ptr()))

    def via_shard(build):
        def run(ix):
            sh = k.shard(ix)
            try:
                build(sh)
            finally:
                sh.close()
        return run

    compare("shard_add", via_shard(lambda sh: sh.add(x, ids)))
    compare("shard_add_device", via_shard(lambda sh: sh.add_device(n, xd.data_ptr(), idd.data_ptr())))

    path = str(tmp_path / f"{kind_name}.idx")
    ref.save(path)
    loaded = k.new(trained=False)
    got = _refusal(lambda: loaded.load(path))
    obs["load"] = got if got != "ok" else ("same" if _same(k.read(loaded), want) else "differs")

    prefix = str(tmp_path / f"{kind_name}.snap")

    def shard_restore():
        sh = k.shard(k.new())  # a row-sharded index is empty when its shard is made
        try:
            sh.add(x, ids)
            sh.save(prefix)
        finally:
            sh.close()
        fresh = k.new(trained=False)
        sh = k.shard(fresh)
        try:
            sh.load(prefix)
        finally:
            sh.close()
        return fresh

    box = []
    got = _refusal(lambda: box.append(shard_restore()))
    obs["shard_load"] = got if got != "ok" else ("same" if _same(k.read(box[0]), want) else "differs")

    src, want_r = ref, want
    if k.hnsw:  # the batched build, alone and through the shard; an HNSW rebuild runs the batched build
        src = k.new()
        src.add_batched(x, ids)
        want_r = k.read(src)
        ix = k.new()
        got = _refusal(lambda: via_shard(lambda sh: sh.hnsw_add_batched(x, ids))(ix))
        obs["shard_add_batched_rows"] = got if got != "ok" else ("same" if _same(k.read(ix), want_r) else "differs")
    rebuilt = k.new(trained=False)
    got = _refusal(lambda: rebuilt.rebuild_from(src))
    obs["rebuild_from"] = got if got != "ok" else ("same" if _same(k.read(rebuilt), want_r) else "differs")

    # upsert of a subset = the other rows, then the subset; on HNSW (an add is an upsert) = the same two adds through the shard
    sub = np.arange(n) % 3 == 0
    keep = k.new()
    if k.hnsw:
        via_shard(lambda sh: (sh.add(x, ids), sh.add(x[sub], ids[sub])))(keep)
    else:
        keep.add(x[~sub], ids[~sub])
        keep.add(x[sub], ids[sub])
    want_u = k.read(keep)

    def upsert_route(route, write_subset):
        ix = k.new()
        ix.add(x, ids)
        got = _refusal(lambda: write_subset(ix))
        obs[route] = got if got != "ok" else ("same" if _same(k.read(ix), want_u) else "differs")

    upsert_route("upsert", lambda ix: ix.upsert(x[sub], ids[sub]))
    xs, ids_s = _dev(x[sub]), _dev(ids[sub])
    upsert_route("upsert_device", lambda ix: ix.add_device(int(sub.sum()), xs.data_ptr(), ids_s.data_ptr(), upsert=True))

    # refusals, each on a fresh index
    L = b200vs.lib()
    two = ids[:2].copy()
    dup = np.array([N + 7, N + 7], dtype=np.int64)  # a new id, twice, into an index that holds rows

    def add_repeated_id():
        ix = k.new()
        ix.add(x[:100], ids[:100])
        ix.add(x[:2], dup)

    obs["add_empty"] = _refusal(lambda: k.new().add(x[:0], ids[:0]))
    obs["add_repeated_id"] = _refusal(add_repeated_id)
    obs["add_untrained"] = _refusal(lambda: k.new(trained=False).add(x[:2], two))
    obs["add_device_untrained"] = _refusal(lambda: k.new(trained=False).add_device(2, xd.data_ptr(), idd.data_ptr()))
    obs["train_after_add"] = _refusal(lambda: ref.train(x))
    obs["add_batched"] = _refusal(lambda: k.new().add_batched(_rows(2, 5), two))
    xf, xb = _rows(2, 6), _bits(2, 6)
    other = k.new()
    if k.binary:
        obs["float_add"] = _refusal(lambda: b200vs._check(L.b200vs_add_with_ids(other.h, 2, xf.ctypes.data, two.ctypes.data, 0)))
        obs["float_train"] = _refusal(lambda: b200vs._check(L.b200vs_train(other.h, 2, xf.ctypes.data)))
    else:
        obs["binary_add"] = _refusal(lambda: b200vs._check(L.b200vs_add_with_ids_binary(other.h, 2, xb.ctypes.data, two.ctypes.data, 0)))
        obs["binary_train"] = _refusal(lambda: b200vs._check(L.b200vs_train_binary(other.h, 2, xb.ctypes.data)))

    # collective adds: a refusal agreed before anything changes leaves the index as it was
    def collective(route, call, ix, rows=0):
        try:
            sh = k.shard(ix)
        except b200vs.B200VSError as e:
            obs[route] = [e.code, e.msg]
            return
        try:
            if rows:
                sh.add(x[:rows], ids[:rows])
            before = ix.get_count()
            obs[route] = _refusal(lambda: call(sh))
        finally:
            sh.close()
        if obs[route] != "ok":
            obs[route].append(ix.get_count() - before)

    collective("shard_add_repeated_id", lambda sh: sh.add(x[:2], dup), k.new(), rows=100)
    if not k.binary:
        collective("shard_add_batched", lambda sh: sh.hnsw_add_batched(_rows(2, 5), two), k.new())
    if k.hnsw:  # max_elements
        small = lambda: k.new(max_elements=100)
        xm, im = _rows(150, 7), np.arange(1, 151, dtype=np.int64)
        obs["add_over_max"] = _refusal(lambda: small().add(xm, im))
        obs["add_batched_over_max"] = _refusal(lambda: small().add_batched(xm, im))
        collective("shard_add_over_max", lambda sh: sh.add(xm, im), small())
        collective("shard_add_batched_over_max", lambda sh: sh.hnsw_add_batched(xm, im), small())
    return obs


KINDS = ["flat_l2", "flat_ip", "flat_cos", "ivf_flat_l2", "ivf_flat_cos", "ivf_pq8_l2", "ivf_pq4_ip", "ivf_pqflat_l2", "hnsw_l2",
         "hnsw_cos", "binary_flat", "binary_ivf"]

# Recorded on the build before every write went through one add request: "same" for a route that builds the index the
# reference route builds, "ok" for a write that is accepted, [status, b200vs_last_error] for one that is refused (and, for
# a collective add, the rows it added: none).
ILL, NOT_TRAIN, NOS, INT, DUP = (b200vs.EILLEGAL_PARAMETERS, b200vs.EVECTOR_NOT_TRAIN, b200vs.EVECTOR_NOT_SUPPORT, b200vs.EINTERNAL,
                                 b200vs.EVECTOR_ID_DUPLICATED)
EXPECTED = {
    "flat_l2": {"add_2": "same", "add_device": [NOS, "device-pointer add only exists for IVF_FLAT and IVF_PQ"],
        "shard_add": "same", "shard_add_device": "same", "load": "same", "shard_load": "same",
        "rebuild_from": [NOS, "a Flat index never needs a rebuild"], "upsert": "same",
        "upsert_device": [NOS, "device-pointer add only exists for IVF_FLAT and IVF_PQ"],
        "add_empty": [ILL, "vector_with_ids is empty"], "add_repeated_id": [DUP, "vector id duplicated: 2007"],
        "add_untrained": "ok", "add_device_untrained": [NOS, "device-pointer add only exists for IVF_FLAT and IVF_PQ"],
        "train_after_add": "ok", "add_batched": [ILL, "batched HNSW construction needs an HNSW index"],
        "binary_add": [ILL, "binary entry point on a float index"],
        "binary_train": [ILL, "binary entry point on a float index"],
        "shard_add_repeated_id": [DUP, "vector id duplicated: 2007", 0],
        "shard_add_batched": [ILL, "batched HNSW construction needs an HNSW index", 0]},
    "flat_ip": {"add_2": "same", "add_device": [NOS, "device-pointer add only exists for IVF_FLAT and IVF_PQ"],
        "shard_add": "same", "shard_add_device": "same", "load": "same", "shard_load": "same",
        "rebuild_from": [NOS, "a Flat index never needs a rebuild"], "upsert": "same",
        "upsert_device": [NOS, "device-pointer add only exists for IVF_FLAT and IVF_PQ"],
        "add_empty": [ILL, "vector_with_ids is empty"], "add_repeated_id": [DUP, "vector id duplicated: 2007"],
        "add_untrained": "ok", "add_device_untrained": [NOS, "device-pointer add only exists for IVF_FLAT and IVF_PQ"],
        "train_after_add": "ok", "add_batched": [ILL, "batched HNSW construction needs an HNSW index"],
        "binary_add": [ILL, "binary entry point on a float index"],
        "binary_train": [ILL, "binary entry point on a float index"],
        "shard_add_repeated_id": [DUP, "vector id duplicated: 2007", 0],
        "shard_add_batched": [ILL, "batched HNSW construction needs an HNSW index", 0]},
    "flat_cos": {"add_2": "same", "add_device": [NOS, "device-pointer add only exists for IVF_FLAT and IVF_PQ"],
        "shard_add": "same", "shard_add_device": "same", "load": "same", "shard_load": "same",
        "rebuild_from": [NOS, "a Flat index never needs a rebuild"], "upsert": "same",
        "upsert_device": [NOS, "device-pointer add only exists for IVF_FLAT and IVF_PQ"],
        "add_empty": [ILL, "vector_with_ids is empty"], "add_repeated_id": [DUP, "vector id duplicated: 2007"],
        "add_untrained": "ok", "add_device_untrained": [NOS, "device-pointer add only exists for IVF_FLAT and IVF_PQ"],
        "train_after_add": "ok", "add_batched": [ILL, "batched HNSW construction needs an HNSW index"],
        "binary_add": [ILL, "binary entry point on a float index"],
        "binary_train": [ILL, "binary entry point on a float index"],
        "shard_add_repeated_id": [DUP, "vector id duplicated: 2007", 0],
        "shard_add_batched": [ILL, "batched HNSW construction needs an HNSW index", 0]},
    "ivf_flat_l2": {"add_2": "same", "add_device": "same", "add_device_lists": "same", "shard_add": "same",
        "shard_add_device": "same", "load": "same", "shard_load": "same", "rebuild_from": "same", "upsert": "same",
        "upsert_device": "same", "add_empty": [ILL, "vector_with_ids is empty"], "add_repeated_id": "ok",
        "add_untrained": [NOT_TRAIN, "not train"], "add_device_untrained": [NOT_TRAIN, "not train"],
        "train_after_add": "ok", "add_batched": [ILL, "batched HNSW construction needs an HNSW index"],
        "binary_add": [ILL, "binary entry point on a float index"],
        "binary_train": [ILL, "binary entry point on a float index"], "shard_add_repeated_id": "ok",
        "shard_add_batched": [ILL, "batched HNSW construction needs an HNSW index", 0]},
    "ivf_flat_cos": {"add_2": "same", "add_device": "same", "add_device_lists": "same", "shard_add": "same",
        "shard_add_device": "same", "load": "same", "shard_load": "same", "rebuild_from": "same", "upsert": "same",
        "upsert_device": "same", "add_empty": [ILL, "vector_with_ids is empty"], "add_repeated_id": "ok",
        "add_untrained": [NOT_TRAIN, "not train"], "add_device_untrained": [NOT_TRAIN, "not train"],
        "train_after_add": "ok", "add_batched": [ILL, "batched HNSW construction needs an HNSW index"],
        "binary_add": [ILL, "binary entry point on a float index"],
        "binary_train": [ILL, "binary entry point on a float index"], "shard_add_repeated_id": "ok",
        "shard_add_batched": [ILL, "batched HNSW construction needs an HNSW index", 0]},
    "ivf_pq8_l2": {"add_2": "same", "add_device": "same", "add_device_lists": "same", "shard_add": "same",
        "shard_add_device": "same", "load": "same", "shard_load": "same",
        "rebuild_from": [NOS, "rebuild_from an IVF_PQ index in IVF-PQ mode: only its codes are stored"], "upsert": "same",
        "upsert_device": "same", "add_empty": [ILL, "vector_with_ids is empty"], "add_repeated_id": "ok",
        "add_untrained": [NOT_TRAIN, "not train"], "add_device_untrained": [NOT_TRAIN, "not train"],
        "train_after_add": "ok", "add_batched": [ILL, "batched HNSW construction needs an HNSW index"],
        "binary_add": [ILL, "binary entry point on a float index"],
        "binary_train": [ILL, "binary entry point on a float index"], "shard_add_repeated_id": "ok",
        "shard_add_batched": [ILL, "batched HNSW construction needs an HNSW index", 0]},
    "ivf_pq4_ip": {"add_2": "same", "add_device": "same", "add_device_lists": "same", "shard_add": "same",
        "shard_add_device": "same", "load": "same", "shard_load": "same",
        "rebuild_from": [NOS, "rebuild_from an IVF_PQ index in IVF-PQ mode: only its codes are stored"], "upsert": "same",
        "upsert_device": "same", "add_empty": [ILL, "vector_with_ids is empty"], "add_repeated_id": "ok",
        "add_untrained": [NOT_TRAIN, "not train"], "add_device_untrained": [NOT_TRAIN, "not train"],
        "train_after_add": "ok", "add_batched": [ILL, "batched HNSW construction needs an HNSW index"],
        "binary_add": [ILL, "binary entry point on a float index"],
        "binary_train": [ILL, "binary entry point on a float index"], "shard_add_repeated_id": "ok",
        "shard_add_batched": [ILL, "batched HNSW construction needs an HNSW index", 0]},
    "ivf_pqflat_l2": {"add_2": "same",
        "add_device": [NOS, "an IVF_PQ index in inner-Flat mode (too few training rows) has no inverted lists"],
        "shard_add": [NOS, "an IVF_PQ index in inner-Flat mode (too few training rows) has no inverted lists to shard"],
        "shard_add_device": [NOS, "an IVF_PQ index in inner-Flat mode (too few training rows) has no inverted lists to shard"],
        "load": "same",
        "shard_load": [NOS, "an IVF_PQ index in inner-Flat mode (too few training rows) has no inverted lists to shard"],
        "rebuild_from": "same", "upsert": "same",
        "upsert_device": [NOS, "an IVF_PQ index in inner-Flat mode (too few training rows) has no inverted lists"],
        "add_empty": [ILL, "vector_with_ids is empty"], "add_repeated_id": [DUP, "vector id duplicated: 2007"],
        "add_untrained": [NOT_TRAIN, "not train"], "add_device_untrained": [NOT_TRAIN, "not train"],
        "train_after_add": "ok", "add_batched": [ILL, "batched HNSW construction needs an HNSW index"],
        "binary_add": [ILL, "binary entry point on a float index"],
        "binary_train": [ILL, "binary entry point on a float index"],
        "shard_add_repeated_id": [NOS, "an IVF_PQ index in inner-Flat mode (too few training rows) has no inverted lists to shard"],
        "shard_add_batched": [NOS, "an IVF_PQ index in inner-Flat mode (too few training rows) has no inverted lists to shard"]},
    "hnsw_l2": {"add_2": "same", "add_device": [NOS, "device-pointer add only exists for IVF_FLAT and IVF_PQ"],
        "shard_add": "same", "shard_add_device": "same", "load": "same", "shard_load": "same", "rebuild_from": "same",
        "shard_add_batched": "ok", "upsert": "same",
        "upsert_device": [NOS, "device-pointer add only exists for IVF_FLAT and IVF_PQ"],
        "add_empty": [ILL, "vector_with_ids is empty"], "add_repeated_id": "ok", "add_untrained": "ok",
        "add_device_untrained": [NOS, "device-pointer add only exists for IVF_FLAT and IVF_PQ"], "train_after_add": "ok",
        "add_batched": "ok", "binary_add": [ILL, "binary entry point on a float index"],
        "binary_train": [ILL, "binary entry point on a float index"], "shard_add_repeated_id": "ok",
        "add_over_max": [INT, "upsert failed, exceeds max elements"],
        "add_batched_over_max": [INT, "upsert failed, exceeds max elements"],
        "shard_add_over_max": [INT, "upsert failed, exceeds max elements", 0],
        "shard_add_batched_over_max": [INT, "upsert failed, exceeds max elements", 0], "shard_add_batched_rows": "same"},
    "hnsw_cos": {"add_2": "same", "add_device": [NOS, "device-pointer add only exists for IVF_FLAT and IVF_PQ"],
        "shard_add": "same", "shard_add_device": "same", "load": "same", "shard_load": "same", "rebuild_from": "same",
        "shard_add_batched": "ok", "upsert": "same",
        "upsert_device": [NOS, "device-pointer add only exists for IVF_FLAT and IVF_PQ"],
        "add_empty": [ILL, "vector_with_ids is empty"], "add_repeated_id": "ok", "add_untrained": "ok",
        "add_device_untrained": [NOS, "device-pointer add only exists for IVF_FLAT and IVF_PQ"], "train_after_add": "ok",
        "add_batched": "ok", "binary_add": [ILL, "binary entry point on a float index"],
        "binary_train": [ILL, "binary entry point on a float index"], "shard_add_repeated_id": "ok",
        "add_over_max": [INT, "upsert failed, exceeds max elements"],
        "add_batched_over_max": [INT, "upsert failed, exceeds max elements"],
        "shard_add_over_max": [INT, "upsert failed, exceeds max elements", 0],
        "shard_add_batched_over_max": [INT, "upsert failed, exceeds max elements", 0], "shard_add_batched_rows": "same"},
    "binary_flat": {"add_2": "same", "add_device": [NOS, "device-pointer add only exists for IVF_FLAT and IVF_PQ"],
        "shard_add": "same", "shard_add_device": "same", "load": "same", "shard_load": "same",
        "rebuild_from": [NOS, "a Flat index never needs a rebuild"], "upsert": "same",
        "upsert_device": [NOS, "device-pointer add only exists for IVF_FLAT and IVF_PQ"],
        "add_empty": [ILL, "vector_with_ids is empty"], "add_repeated_id": [DUP, "vector id duplicated: 2007"],
        "add_untrained": "ok", "add_device_untrained": [NOS, "device-pointer add only exists for IVF_FLAT and IVF_PQ"],
        "train_after_add": "ok", "add_batched": [ILL, "batched HNSW construction needs an HNSW index"],
        "float_add": [ILL, "float entry point on a binary index"],
        "float_train": [ILL, "float entry point on a binary index"],
        "shard_add_repeated_id": [DUP, "vector id duplicated: 2007", 0]},
    "binary_ivf": {"add_2": "same", "add_device": [NOS, "device-pointer add only exists for IVF_FLAT and IVF_PQ"],
        "shard_add": "same", "shard_add_device": "same", "load": "same", "shard_load": "same", "rebuild_from": "same",
        "upsert": "same", "upsert_device": [NOS, "device-pointer add only exists for IVF_FLAT and IVF_PQ"],
        "add_empty": [ILL, "vector_with_ids is empty"], "add_repeated_id": "ok", "add_untrained": [NOT_TRAIN, "not train"],
        "add_device_untrained": [NOS, "device-pointer add only exists for IVF_FLAT and IVF_PQ"], "train_after_add": "ok",
        "add_batched": [ILL, "batched HNSW construction needs an HNSW index"],
        "float_add": [ILL, "float entry point on a binary index"],
        "float_train": [ILL, "float entry point on a binary index"], "shard_add_repeated_id": "ok"},
}


@pytest.mark.parametrize("kind", KINDS)
def test_write_routes(kind, tmp_path):
    assert observe(kind, tmp_path) == EXPECTED[kind]
