"""Row lifecycle of every row-store index, checked against a numpy model of its rows after every write.

The model holds each inverted list's rows in storage order as (id, stored row); a Flat index has one list.  It restates the
semantics the indexes document:
  - Flat, Binary Flat and IVF-PQ in inner-Flat mode: add and upsert are one operation (rows holding the batch's ids are
    removed, the new rows are appended at the end); a batch with a repeated id is refused with EVECTOR_ID_DUPLICATED and
    changes nothing; a delete ignores unknown ids and returns how many rows it removed.
  - IVF-Flat, IVF-PQ and Binary IVF-Flat: an add appends each row at the tail of its list (the nearest list of a host add,
    the caller's list of a device add with lists, which need not be the nearest); a repeated id, in the batch or already
    in the index, becomes another row; an upsert first removes every row holding its ids; a delete removes every row
    holding its ids, and one that removes nothing is refused with EVECTOR_INVALID.
Cosine rows are stored as oracle.normalize_faiss(x); IVF-PQ rows as the oracle encoder's codes of the model's rows in the
model's lists.  Trained states are fixed with the state blobs, so the model knows the centroids and codebooks exactly.

Seeded histories mix adds of 1 to 2 500 rows (some gathered around one centroid, so one list is relocated again and again;
some through the device add with and without the caller's lists), upserts, deletes of present, absent and repeated ids,
whole-list and whole-index deletes, and save then load into a fresh index, after which the history goes on writing on the
loaded index.  After every step: the live count, export_lists (offsets, ids in order, rows bit for bit), reconstruct on a
float Flat index, search against the oracle run on the model's own lists (the tile path, exact_only and a batch of 5; all
lists and a few lists on IVF), and the bookkeeping bounds (Flat: fewer tombstones than live rows; IVF: tombstones at most
max(live rows, 4096), the compaction threshold).

Targeted cases: an IVF upsert-only workload stays compact, the exact rows at which Flat and IVF compaction starts, and a
negative id refused by every add route before anything changes."""
import zlib

import numpy as np
import pytest

import b200vs
import binary_oracle
import pq_codes
from b200vs import BINARY_FLAT, BINARY_IVF_FLAT, COSINE, FLAT, HAMMING, HNSW, IP, IVF_FLAT, IVF_PQ, L2
from gpu_util import assert_same_results, require_gpu

pytestmark = pytest.mark.gpu
NLIST, K, BITS, PQ_M, PQ_D, FLOAT_D, COS_D = 16, 20, 256, 8, 32, 64, 36
IVF_COMPACT_MIN = 4096  # IvfLists::compact_if_needed: garbage + tombstones must exceed max(live rows, 4096)
SIZES, SIZE_P = np.array([1, 7, 300, 2500]), [0.15, 0.15, 0.3, 0.4]
ABSENT = 10 ** 12  # ids from here up are never added


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


class Kind:
    """One index kind: how to make it, its rows, its model's expected export and its oracle search."""

    def __init__(self, name, o):
        self.name, self.o = name, o
        self.binary = name.startswith("binary")
        self.pqflat = name == "ivf_pqflat_l2"
        self.pq = name.startswith(("ivf_pq8", "ivf_pq4"))
        self.ivf = name.startswith("ivf_flat") or self.pq or name == "binary_ivf"
        self.float_flat = name.startswith("flat")
        self.device_adds = self.ivf and not self.binary  # b200vs_add_with_ids_device: IVF_FLAT and IVF_PQ
        self.nlist = NLIST if self.ivf else 1
        self.nbits = 4 if name.startswith("ivf_pq4") else 8
        self.metric = HAMMING if self.binary else {"l2": L2, "ip": IP, "cos": COSINE}[name.split("_")[-1]]
        self.d = BITS if self.binary else PQ_D if (self.pq or self.pqflat) else COS_D if name == "ivf_flat_cos" else FLOAT_D
        self.cs = pq_codes.code_size(PQ_M, self.nbits)
        rng = np.random.default_rng(zlib.crc32(name.encode()))
        self.blob = None
        if name == "binary_ivf":
            self.cent = rng.integers(0, 256, (NLIST, BITS // 8), dtype=np.uint8)
            self.blob = b200vs.binary_ivf_state_blob(self.cent)
        elif self.ivf:
            self.cent = self.stored(rng.standard_normal((NLIST, self.d)).astype(np.float32))
            if self.pq:
                self.cb = (0.5 * rng.standard_normal((PQ_M, 1 << self.nbits, self.d // PQ_M))).astype(np.float32)
                self.blob = b200vs.ivfpq_state_blob(self.cent, self.cb, self.metric)
            else:
                self.blob = b200vs.ivf_state_blob(self.cent, self.metric)
        self.q = self.rows(np.random.default_rng(7), 64)

    def new(self, trained=True):
        if self.binary:
            ix = b200vs.Index(BINARY_FLAT if self.name == "binary_flat" else BINARY_IVF_FLAT, HAMMING, BITS, nlist=NLIST)
        elif self.float_flat:
            ix = b200vs.Index(FLAT, self.metric, self.d)
        elif self.name.startswith("ivf_flat"):
            ix = b200vs.Index(IVF_FLAT, self.metric, self.d, nlist=NLIST)
        else:
            ix = b200vs.Index(IVF_PQ, self.metric, self.d, nlist=NLIST, pq_m=PQ_M, pq_nbits=self.nbits)
        if trained and self.blob is not None:
            ix.set_trained_state(self.blob)
        elif trained and self.pqflat:
            ix.train(np.random.default_rng(3).standard_normal((100, self.d)).astype(np.float32))  # too few rows: inner Flat
            assert ix.sub_type() == FLAT
        return ix

    def rows(self, rng, n, around=None):
        """n raw rows; around = a list whose centroid they gather near."""
        if self.binary:
            if around is None or self.name == "binary_flat":
                return rng.integers(0, 256, (n, BITS // 8), dtype=np.uint8)
            x = np.repeat(self.cent[around:around + 1], n, axis=0)
            for _ in range(8):
                bit = rng.integers(0, BITS, n)
                x[np.arange(n), bit >> 3] ^= (1 << (bit & 7)).astype(np.uint8)
            return x
        x = rng.standard_normal((n, self.d)).astype(np.float32)
        if around is not None and self.ivf:
            x = (3 * self.cent[around] + 0.3 * x).astype(np.float32)
        return x

    def stored(self, x):
        return self.o.normalize_faiss(x) if self.metric == COSINE else x

    def assign(self, stored):
        if self.name == "binary_ivf":
            return binary_oracle.assign(stored, self.cent).astype(np.int64)
        return self.o.assign(self.metric, stored, self.cent).astype(np.int64)

    def model(self):
        if self.binary:
            return Model(self.nlist, (BITS // 8,), np.uint8)
        return Model(self.nlist, (self.d,), np.float32)

    def export(self, ix):
        """(offsets, ids, rows) of ix: float rows, packed bits, or PQ code rows."""
        if self.pq:
            off, _, codes, ids = ix.export_lists(self.nlist, with_vectors=False, code_size=self.cs)
            return off, ids, codes
        off, vec, codes, ids = ix.export_lists(self.nlist)
        return off, ids, codes if self.binary else vec

    def expected(self, m):
        """(offsets, ids, rows) the model holds, in export form."""
        off, ids, rows = m.export()
        if self.pq:
            lists = np.repeat(np.arange(self.nlist), np.diff(off))
            rows = pq_codes.ivfpq_encode(self.o, self.cb, self.cent, rows, lists) if len(ids) else np.zeros((0, self.cs), np.uint8)
        return off, ids, rows

    def oracle_search(self, exp, xq, nprobe):
        off, ids, rows = exp
        if self.name == "binary_flat":
            return binary_oracle.flat_search(rows, ids, xq, K)
        if self.name == "binary_ivf":
            return binary_oracle.ivf_search(self.cent, off, rows, ids, xq, K, nprobe)
        if self.pq:
            return pq_codes.ivfpq_search(self.o, self.metric, self.cent, self.cb, off, rows, ids, xq, K, nprobe, nthreads=8)
        if self.ivf:
            return self.o.ivfflat_search(self.metric, self.cent, off, rows, ids, xq, K, nprobe, nthreads=8)
        return self.o.flat_search(self.metric, rows, ids, xq, K, nthreads=8)

    def check(self, ix, m, where, reconstruct_rng=None, never=None):
        """Every check of one state of ix against the model m."""
        n = m.count()
        assert ix.get_count() == n, f"{where}: count {ix.get_count()} != model {n}"
        exp = self.expected(m)
        off, ids, rows = self.export(ix)
        assert np.array_equal(off, exp[0]), f"{where}: list offsets differ from the model"
        assert np.array_equal(ids, exp[1]), f"{where}: ids differ from the model (storage order)"
        assert rows.shape == exp[2].shape and np.array_equal(rows.view(np.uint8), exp[2].view(np.uint8)), f"{where}: rows differ from the model"
        if self.float_flat and reconstruct_rng is not None:
            live = exp[1]
            pick = reconstruct_rng.choice(live.size, min(live.size, 64), replace=False) if live.size else np.zeros(0, np.int64)
            gone = np.array(sorted(never), np.int64) if never else np.zeros(0, np.int64)
            ask = np.concatenate([live[pick], gone[:32], ABSENT + np.arange(3)])
            out, found = ix.reconstruct(ask)
            assert found[:pick.size].all() and not found[pick.size:].any(), f"{where}: reconstruct found the wrong ids"
            assert np.array_equal(out[:pick.size].view(np.uint32), exp[2][pick].view(np.uint32)), f"{where}: reconstruct rows differ"
        for nprobe in ((self.nlist, 3) if self.ivf else (0,)):
            for xq, exact in ((self.q, False), (self.q, True), (self.q[:5], False)):
                kw = dict(exact_only=exact)
                if self.ivf:
                    kw["nprobe"] = nprobe
                Dg, Ig = ix.search(xq, K, **kw)
                Do, Io = self.oracle_search(exp, xq, nprobe)
                try:
                    assert_same_results(Dg, Ig, Do, Io)
                except AssertionError as e:
                    raise AssertionError(f"{where}: search nq={len(xq)} exact_only={exact} nprobe={nprobe}: {e}") from None
        dc = ix.get_deleted_count()
        if self.ivf:
            assert dc <= max(n, IVF_COMPACT_MIN), f"{where}: {dc} tombstones beside {n} live rows"
        else:
            assert dc == 0 or 2 * dc < n + dc, f"{where}: {dc} tombstones beside {n} live rows"


class Model:
    """Each list's (ids, stored rows) in storage order."""

    def __init__(self, nlist, row_shape, dtype):
        self.ids = [np.zeros(0, np.int64) for _ in range(nlist)]
        self.rows = [np.zeros((0,) + row_shape, dtype) for _ in range(nlist)]

    def count(self):
        return sum(i.size for i in self.ids)

    def live(self):
        return np.unique(np.concatenate(self.ids))

    def append(self, lists, ids, rows):
        for l in np.unique(lists):
            sel = lists == l
            self.ids[l] = np.concatenate([self.ids[l], ids[sel]])
            self.rows[l] = np.concatenate([self.rows[l], rows[sel]])

    def remove(self, ids):
        """Drop every row holding one of ids; returns how many."""
        n = 0
        for l in range(len(self.ids)):
            keep = ~np.isin(self.ids[l], ids)
            n += int(keep.size - keep.sum())
            self.ids[l], self.rows[l] = self.ids[l][keep], self.rows[l][keep]
        return n

    def export(self):
        off = np.concatenate([[0], np.cumsum([i.size for i in self.ids])]).astype(np.int64)
        return off, np.concatenate(self.ids), np.concatenate(self.rows)


class History:
    """A seeded history of writes on one index, mirrored on the model and checked after every step."""

    def __init__(self, kind, rng, tmp_path, reserve=False):
        self.k, self.rng, self.tmp = kind, rng, tmp_path
        self.ix = kind.new()
        self.m = kind.model()
        self.next_id = 1
        self.gone = set()  # ids added once and deleted since
        self.compactions = 0
        self.tombstoned = 0  # rows the current step turned into tombstones
        self.peak = 0
        if reserve:
            self.ix.reserve_lists(np.full(NLIST, 400, np.int64))

    def fresh(self, n):
        ids = np.arange(self.next_id, self.next_id + n, dtype=np.int64)
        self.next_id += n
        return ids

    def present(self, n):
        live = self.m.live()
        return self.rng.choice(live, min(n, live.size), replace=False) if live.size else np.zeros(0, np.int64)

    def write(self, x, ids, upsert=False, route="host", lists=None):
        k, m = self.k, self.m
        stored = k.stored(x)
        if k.ivf:
            if upsert:
                self.tombstoned += m.remove(ids)
            m.append(lists if lists is not None else k.assign(stored), ids, stored)
        else:
            self.tombstoned += m.remove(ids)
            m.append(np.zeros(len(ids), np.int64), ids, stored)
        self.gone -= set(ids.tolist())
        if route == "host":
            self.ix.add(x, ids, upsert=upsert)
        else:
            xd, idd = _dev(x), _dev(ids)
            ld = _dev(lists) if lists is not None else None
            self.ix.add_device(len(ids), xd.data_ptr(), idd.data_ptr(), ld.data_ptr() if ld is not None else None, upsert=upsert)

    def delete(self, ids):
        before = set(self.m.live().tolist())
        want = self.m.remove(ids)
        self.tombstoned += want
        self.gone |= before - set(self.m.live().tolist())
        if self.k.ivf and want == 0:
            with pytest.raises(b200vs.B200VSError) as e:
                self.ix.delete(ids)
            assert e.value.code == b200vs.EVECTOR_INVALID
        else:
            assert self.ix.delete(ids) == want

    def add_step(self, upsert):
        rng, k = self.rng, self.k
        n = int(rng.choice(SIZES, p=SIZE_P))
        if upsert:
            p = int(rng.integers(0, n + 1))
            ids = np.concatenate([self.present(p), self.fresh(n)])[:n]
        else:
            ids = self.fresh(n)
            if rng.random() < 0.2:  # ids already present: replaced on a Flat index, another row on an IVF index
                old = self.present(int(rng.integers(1, n + 1)))
                ids[:old.size] = old
        ids = rng.permutation(ids)
        x = k.rows(rng, n, around=int(rng.integers(k.nlist)) if rng.random() < 0.3 else None)
        route, lists = "host", None
        if k.device_adds and rng.random() < 0.35:
            route = "device"
            if rng.random() < 0.5:  # the caller's lists, not the nearest ones
                lists = rng.integers(0, k.nlist, n).astype(np.int64)
        self.write(x, ids, upsert=upsert, route=route, lists=lists)
        return f"{'upsert' if upsert else 'add'} {n} via {route}{' with lists' if lists is not None else ''}"

    def delete_step(self):
        rng = self.rng
        live = self.m.live()
        p = int(rng.integers(0, max(1, live.size // 3) + 1))
        ids = self.present(p)
        extra = [ABSENT + rng.integers(0, 1000, int(rng.integers(0, 20))), np.array(sorted(self.gone)[:5], np.int64)]
        if ids.size:
            extra.append(rng.choice(ids, int(rng.integers(0, 5))))  # repeated in the batch
        ids = rng.permutation(np.concatenate([ids] + extra).astype(np.int64))
        self.delete(ids)
        return f"delete {ids.size} ids"

    def delete_list_step(self):
        k = self.k
        if k.ivf:
            full = [l for l in range(k.nlist) if self.m.ids[l].size]
            if not full:
                return self.add_step(False)
            l = int(self.rng.choice(full))
            self.delete(np.unique(self.m.ids[l]))
            return f"delete list {l}"
        ids = self.m.ids[0]  # a Flat index: one block of rows in storage order
        a = int(self.rng.integers(0, max(1, ids.size)))
        self.delete(ids[a:a + int(self.rng.integers(1, 3000))])
        return "delete a block"

    def delete_all_step(self):
        live = self.m.live()
        if not live.size:
            return self.add_step(False)
        self.delete(self.rng.permutation(live))
        return "delete everything"

    def reload_step(self):
        path = str(self.tmp / f"{self.k.name}.{self.next_id}.idx")
        self.ix.save(path)
        fresh = self.k.new(trained=False)
        fresh.load(path)
        self.ix.close()
        self.ix = fresh
        return "save + load"

    def repeated_step(self):
        """A batch with an id twice: refused on a Flat index (nothing changes), two rows on an IVF index."""
        n = int(self.rng.choice(SIZES[1:3]))
        ids = self.fresh(n)
        ids[-1] = ids[0]
        x = self.k.rows(self.rng, n)
        if self.k.ivf:
            self.write(x, ids)
        else:
            with pytest.raises(b200vs.B200VSError) as e:
                self.ix.add(x, ids)
            assert e.value.code == b200vs.EVECTOR_ID_DUPLICATED
        return "repeated id"

    def run(self, steps):
        for s in range(steps):
            r = self.rng.random()
            dc = self.ix.get_deleted_count()
            self.tombstoned = 0
            if r < 0.40 or self.m.count() == 0:
                what = self.add_step(False)
            elif r < 0.56:
                what = self.add_step(True)
            elif r < 0.78:
                what = self.delete_step()
            elif r < 0.84:
                what = self.delete_list_step()
            elif r < 0.87:
                what = self.delete_all_step()
            elif r < 0.94:
                what = self.reload_step()
            else:
                what = self.repeated_step()
            if self.ix.get_deleted_count() < dc + self.tombstoned and "load" not in what:  # the step ended in a compaction
                self.compactions += 1
            self.peak = max(self.peak, self.m.count())
            self.k.check(self.ix, self.m, f"{self.k.name} step {s} ({what}, {self.m.count()} rows)", self.rng, self.gone)


KINDS = ["flat_l2", "flat_cos", "flat_ip", "ivf_flat_l2", "ivf_flat_cos", "ivf_flat_ip", "ivf_pq8_l2", "ivf_pq4_ip",
         "ivf_pqflat_l2", "binary_flat", "binary_ivf"]
IVF_KINDS = ["ivf_flat_l2", "ivf_flat_cos", "ivf_flat_ip", "ivf_pq8_l2", "ivf_pq4_ip", "binary_ivf"]
RESERVABLE = [k for k in IVF_KINDS if k != "binary_ivf"]  # b200vs_reserve_lists: IVF_FLAT and IVF_PQ


@pytest.mark.parametrize("kind,reserve", [(k, False) for k in KINDS] + [(k, True) for k in RESERVABLE])
def test_history_matches_model(oracle, tmp_path, kind, reserve):
    k = Kind(kind, oracle)
    h = History(k, np.random.default_rng(zlib.crc32(f"{kind}/{reserve}".encode())), tmp_path, reserve=reserve)
    h.run(80)
    assert h.peak >= 6000, f"the history never held more than {h.peak} live rows"
    assert h.compactions >= 2, f"the history compacted the index only {h.compactions} times (at most {h.peak} live rows)"


@pytest.mark.parametrize("kind", IVF_KINDS)
def test_upsert_loop_stays_compact(oracle, kind):
    """The same 5 000 ids upserted 40 times: tombstones and relocation garbage are compacted away as a delete's are."""
    k = Kind(kind, oracle)
    rng = np.random.default_rng(11)
    ix, m = k.new(), k.model()
    ids = np.arange(1, 5001, dtype=np.int64)
    x = k.rows(rng, ids.size)
    m.append(k.assign(k.stored(x)), ids, k.stored(x))
    ix.add(x, ids)
    mem = {}
    for r in range(1, 41):
        x = k.rows(rng, ids.size)
        m.remove(ids)
        m.append(k.assign(k.stored(x)), ids, k.stored(x))
        ix.upsert(x, ids)
        assert ix.get_count() == ids.size
        dc = ix.get_deleted_count()
        assert dc <= max(ix.get_count(), IVF_COMPACT_MIN), f"round {r}: {dc} tombstones beside {ix.get_count()} live rows"
        mem[r] = ix.get_memory_size()
    assert mem[40] <= 2 * mem[2], f"memory grew from {mem[2]} B after round 2 to {mem[40]} B after round 40"
    k.check(ix, m, f"{kind} after 40 upsert rounds")


@pytest.mark.parametrize("kind", ["flat_l2", "binary_flat"])
def test_flat_compaction_boundary(oracle, kind):
    """2N rows: N - 1 tombstones stay, the N-th compacts."""
    k = Kind(kind, oracle)
    N = 2000
    rng = np.random.default_rng(5)
    ix, m = k.new(), k.model()
    ids = np.arange(1, 2 * N + 1, dtype=np.int64)
    x = k.rows(rng, ids.size)
    ix.add(x, ids)
    m.append(np.zeros(ids.size, np.int64), ids, k.stored(x))
    dead = rng.permutation(ids)[:N]
    assert ix.delete(dead[:N - 1]) == m.remove(dead[:N - 1]) == N - 1
    assert ix.get_deleted_count() == N - 1
    k.check(ix, m, f"{kind}: N - 1 tombstones")
    assert ix.delete(dead[N - 1:]) == m.remove(dead[N - 1:]) == 1
    assert ix.get_deleted_count() == 0 and ix.get_count() == N
    k.check(ix, m, f"{kind}: compacted")


@pytest.mark.parametrize("kind", RESERVABLE)
def test_ivf_compaction_boundary(oracle, kind):
    """Reserved lists (no relocation garbage) and 10 000 rows: 5 000 tombstones stay, the 5 001st compacts, and the export
    and search are what they were before the compaction."""
    k = Kind(kind, oracle)
    rng = np.random.default_rng(6)
    ix, m = k.new(), k.model()
    ids = np.arange(1, 10001, dtype=np.int64)
    x = k.rows(rng, ids.size)
    lists = k.assign(k.stored(x))
    ix.reserve_lists(np.bincount(lists, minlength=NLIST).astype(np.int64))
    ix.add(x, ids)
    m.append(lists, ids, k.stored(x))
    dead = rng.permutation(ids)[:5001]
    assert ix.delete(dead[:5000]) == m.remove(dead[:5000]) == 5000
    assert ix.get_deleted_count() == 5000
    k.check(ix, m, f"{kind}: 5000 tombstones")
    assert ix.delete(dead[5000:]) == m.remove(dead[5000:]) == 1
    assert ix.get_deleted_count() == 0 and ix.get_count() == 4999
    k.check(ix, m, f"{kind}: compacted")


NEG_KINDS = KINDS + ["hnsw_l2"]


@pytest.mark.parametrize("kind", NEG_KINDS)
@pytest.mark.parametrize("bad", [-1, -7])
def test_negative_id_refused(oracle, kind, bad):
    """A batch valid but for one negative id is refused by every add route of the kind before anything changes."""
    rng = np.random.default_rng(-bad)
    if kind == "hnsw_l2":
        k = None
        ix = b200vs.Index(HNSW, L2, 32, hnsw_m=16, hnsw_efc=64, max_elements=2000)
        rows = lambda n: rng.standard_normal((n, 32)).astype(np.float32)
        state = lambda: [ix.get_count(), ix.get_memory_size()] + [a.tobytes() for a in ix.export_lists(1) if a is not None]
    else:
        k = Kind(kind, oracle)
        ix = k.new()
        rows = lambda n: k.rows(rng, n)
        state = lambda: [ix.get_count(), ix.get_memory_size()] + [a.tobytes() for a in k.export(ix)]
    sh = None
    if kind != "ivf_pqflat_l2":  # inner-Flat mode has no lists to shard; a row-sharded index must be empty here
        sh = (b200vs.BinaryShard if kind.startswith("binary") else b200vs.Shard)(ix, 0, 1, None)
    ix.add(rows(300), np.arange(1, 301, dtype=np.int64))
    x, ids = rows(50), np.arange(100001, 100051, dtype=np.int64)
    ids[25] = bad
    want = [b200vs.EILLEGAL_PARAMETERS, f"vector id is negative: {bad}"]
    before = state()
    routes = {"add": lambda: ix.add(x, ids), "upsert": lambda: ix.upsert(x, ids)}
    if k is not None and k.device_adds:
        xd, idd, ld = _dev(x), _dev(ids), _dev(np.zeros(len(ids), np.int64))
        routes["add_device"] = lambda: ix.add_device(len(ids), xd.data_ptr(), idd.data_ptr())
        routes["add_device_lists"] = lambda: ix.add_device(len(ids), xd.data_ptr(), idd.data_ptr(), ld.data_ptr())
        routes["upsert_device"] = lambda: ix.add_device(len(ids), xd.data_ptr(), idd.data_ptr(), upsert=True)
    if kind == "hnsw_l2":
        routes["add_batched"] = lambda: ix.add_batched(x, ids)
    if sh is not None:
        routes["shard_add"] = lambda: sh.add(x, ids)
    try:
        for route, call in routes.items():
            with pytest.raises(b200vs.B200VSError) as e:
                call()
            assert [e.value.code, e.value.msg] == want, f"{kind} {route}"
            assert state() == before, f"{kind} {route}: the refused batch changed the index"
    finally:
        if sh is not None:
            sh.close()


@pytest.mark.parametrize("metric", [L2, IP, COSINE])
def test_negative_id_refused_by_scan(metric):
    """The streaming top-k scan, which adds each tile to a Flat index, refuses a tile with a negative id and keeps the
    results of the tiles before it.  (The range scan stores no rows: it skips negative ids, test_gpu_scan_range.py.)"""
    rng = np.random.default_rng(metric)
    xq = rng.standard_normal((8, 32)).astype(np.float32)
    good, ids = rng.standard_normal((500, 32)).astype(np.float32), np.arange(1, 501, dtype=np.int64)
    bad_ids = np.arange(1001, 1101, dtype=np.int64)
    bad_ids[40] = -7
    bad = rng.standard_normal((100, 32)).astype(np.float32)
    want = [b200vs.EILLEGAL_PARAMETERS, "vector id is negative: -7"]
    ref = b200vs.BruteForceScan(metric, 32, xq, 10)
    ref.push(good, ids)
    want_out = ref.finish()
    s = b200vs.BruteForceScan(metric, 32, xq, 10)
    s.push(good, ids)
    with pytest.raises(b200vs.B200VSError) as e:
        s.push(bad, bad_ids)
    assert [e.value.code, e.value.msg] == want
    for a, b in zip(s.finish(), want_out):
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8))
