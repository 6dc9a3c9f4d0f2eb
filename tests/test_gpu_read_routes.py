"""Every read entry point of every index type, on small seeded indexes (one GPU).

One index kind at a time: the host search at nq = 1 and nq = 64, b200vs_search_device, b200vs_coarse_device followed by
b200vs_search_probes_device, the host range search, and the sharded top-k and range calls at a world of one, where the
type has them.  Routes that answer the same question must give the same ids, distance bits and counts.  Each route's
stats()[0] (kernels launched) and stats()[1] (queries on the tile scan) must equal the recorded values, and every
refused (type, entry point) pair must return the recorded status code and b200vs_last_error text."""
import numpy as np
import pytest

import b200vs
from b200vs import BINARY_FLAT, BINARY_IVF_FLAT, COSINE, FLAT, HAMMING, HNSW, IP, IVF_FLAT, IVF_PQ, L2
from gpu_util import require_gpu

pytestmark = pytest.mark.gpu
D, BITS, NLIST, NPROBE, K, MR, N = 32, 256, 16, 6, 10, 64, 3000
NAN = float("nan")


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def _rows(n, seed, d=D):
    return np.random.default_rng(seed).standard_normal((n, d)).astype(np.float32)


def _bits(n, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, BITS // 8), dtype=np.uint8)


def _make(kind):
    """(index, queries [64, row], shard at a world of one or None) of one kind, with N rows of ids 1..N.  A row-sharded
    index (FLAT, HNSW) gets its shard while it is empty and its rows through it."""
    ids = np.arange(1, N + 1, dtype=np.int64)
    if kind.startswith("binary"):
        ix = b200vs.Index(BINARY_FLAT if kind == "binary_flat" else BINARY_IVF_FLAT, HAMMING, BITS, nlist=NLIST)
        ix.train(_bits(N, 1))
        ix.add(_bits(N, 1), ids)
        return ix, _bits(64, 2), None
    metric = {"l2": L2, "ip": IP, "cos": COSINE}[kind.split("_")[-1]]
    if kind.startswith("flat"):
        ix = b200vs.Index(FLAT, metric, D)
    elif kind.startswith("ivf_flat"):
        ix = b200vs.Index(IVF_FLAT, metric, D, nlist=NLIST)
        ix.train(_rows(N, 1))
    elif kind.startswith("hnsw"):
        ix = b200vs.Index(HNSW, metric, D, hnsw_m=16, hnsw_efc=100, max_elements=2 * N)
    else:  # ivf_pq8 / ivf_pq4: the IVF-PQ mode; ivf_pqflat: too few training rows, the inner Flat index
        nbits = {"ivf_pq8": 8, "ivf_pq4": 4, "ivf_pqflat": 8}[kind.rsplit("_", 1)[0]]
        ix = b200vs.Index(IVF_PQ, metric, D, nlist=NLIST, pq_m=8, pq_nbits=nbits)
        ix.train(_rows(100 if "flat" in kind else max(256 * NLIST, 256 << nbits) + 1000, 3))
        assert ix.sub_type() == (FLAT if "flat" in kind else IVF_PQ)
    if kind.startswith(("flat", "hnsw")):
        sh = b200vs.Shard(ix, 0, 1, None)
        sh.add(_rows(N, 1), ids)
        return ix, _rows(64, 2), sh
    ix.add(_rows(N, 1), ids)
    return ix, _rows(64, 2), None


def _refusal(call):
    with pytest.raises(b200vs.B200VSError) as e:
        call()
    return [e.value.code, e.value.msg]


def _same(a, b):
    for x, y in zip(a, b):
        x, y = np.asarray(x), np.asarray(y)
        assert x.shape == y.shape and np.array_equal(x.view(np.uint8), y.view(np.uint8))


def observe(kind):
    """{route: [stats()[0], stats()[1]] or [status, last_error]} of one index kind; equivalent routes checked equal."""
    import torch

    ix, xq, sh = _make(kind)
    ix.coalescing(0)
    nq = xq.shape[0]
    binary, ivf = kind.startswith("binary"), kind.startswith(("ivf_flat", "ivf_pq8", "ivf_pq4"))
    obs = {}

    def note(route):
        obs[route] = ix.stats()[:2]

    sp, _keep = b200vs.make_search_params(nprobe=NPROBE)
    host = ix.search(xq, K, nprobe=NPROBE)
    note("search_64")
    one = ix.search(xq[:1], K, nprobe=NPROBE)
    note("search_1")
    _same(one, (host[0][:1], host[1][:1]))

    qd = torch.from_numpy(xq).cuda()
    od = torch.empty((nq, K), dtype=torch.float32, device="cuda")
    oi = torch.empty((nq, K), dtype=torch.int64, device="cuda")
    ix.search_device(nq, qd.data_ptr(), K, od.data_ptr(), oi.data_ptr(), sp=sp)
    note("search_device")
    _same(host, (od.cpu().numpy(), oi.cpu().numpy()))

    score = torch.empty((nq, NPROBE), dtype=torch.float32, device="cuda")
    lists = torch.empty((nq, NPROBE), dtype=torch.int64, device="cuda")
    coarse = lambda: ix.coarse_device(nq, qd.data_ptr(), NPROBE, 0, NLIST, score.data_ptr(), lists.data_ptr())
    probed = lambda: ix.search_probes_device(nq, qd.data_ptr(), K, lists.data_ptr(), NPROBE, od.data_ptr(), oi.data_ptr(), sp=sp)
    if ivf:
        coarse()
        note("coarse_device")
        od.zero_()
        probed()
        note("search_probes_device")
        _same(host, (od.cpu().numpy(), oi.cpu().numpy()))
    else:
        lists.zero_()
        obs["coarse_device"] = _refusal(coarse)
        obs["search_probes_device"] = _refusal(probed)

    radius = float(np.median(host[0][:, K // 2]))
    if kind.startswith("hnsw"):
        obs["range_search"] = _refusal(lambda: ix.range_search(xq, radius, MR, nprobe=NPROBE))
    else:
        rng = ix.range_search(xq, radius, MR, nprobe=NPROBE)
        note("range_search")
        assert rng[2].sum() > 0
        if binary:
            obs["range_search_nan"] = _refusal(lambda: ix.range_search(xq, NAN, MR, nprobe=NPROBE))
        else:
            Dn, In, Cn = ix.range_search(xq, NAN, MR, nprobe=NPROBE)
            note("range_search_nan")
            assert not Cn.any() and (In == -1).all() and not Dn.any()

    if not binary:
        try:
            sh = sh or b200vs.Shard(ix, 0, 1, None)
        except b200vs.B200VSError as e:
            obs["shard"] = [e.code, e.msg]
            return obs
        try:
            if kind == "ivf_pqflat":
                obs["shard_search"] = _refusal(lambda: sh.search(xq, K, nprobe=NPROBE))
                return obs
            _same(sh.search(xq, K, nprobe=NPROBE), host)
            note("shard_search")
            if kind.startswith("hnsw"):
                obs["shard_range_search"] = _refusal(lambda: sh.range_search(xq, radius, MR, nprobe=NPROBE))
            else:
                _same(sh.range_search(xq, radius, MR, nprobe=NPROBE), rng)
                note("shard_range_search")
                _same(sh.range_search(xq, NAN, MR, nprobe=NPROBE), (Dn, In, Cn))
                note("shard_range_search_nan")
        finally:
            sh.close()
    return obs


KINDS = ["flat_l2", "flat_ip", "flat_cos", "ivf_flat_l2", "ivf_flat_cos", "ivf_pq8_l2", "ivf_pq4_ip", "ivf_pqflat_l2", "hnsw_l2",
         "hnsw_cos", "binary_flat", "binary_ivf"]

# Recorded on the build before every read went through one search request: [stats()[0], stats()[1]] of a route that
# answers, [status, b200vs_last_error] of one that is refused.  (IVF-PQ in inner-Flat mode copies the inner index's
# counters after a top-k search, which add up over calls, and none after a range search.)
ILL, NOS = b200vs.EILLEGAL_PARAMETERS, b200vs.EVECTOR_NOT_SUPPORT
EXPECTED = {
    "flat_l2": {"search_64": [13, 64], "search_1": [2, 0], "search_device": [13, 64],
        "coarse_device": [NOS, "coarse quantiser only exists for IVF_FLAT and IVF_PQ"],
        "search_probes_device": [NOS, "probe-driven search only exists for IVF_FLAT and IVF_PQ"], "range_search": [12, 64],
        "range_search_nan": [0, 0], "shard_search": [16, 64], "shard_range_search": [16, 64],
        "shard_range_search_nan": [4, 0]},
    "flat_ip": {"search_64": [13, 64], "search_1": [2, 0], "search_device": [13, 64],
        "coarse_device": [NOS, "coarse quantiser only exists for IVF_FLAT and IVF_PQ"],
        "search_probes_device": [NOS, "probe-driven search only exists for IVF_FLAT and IVF_PQ"], "range_search": [12, 64],
        "range_search_nan": [0, 0], "shard_search": [17, 64], "shard_range_search": [16, 64],
        "shard_range_search_nan": [4, 0]},
    "flat_cos": {"search_64": [14, 64], "search_1": [3, 0], "search_device": [14, 64],
        "coarse_device": [NOS, "coarse quantiser only exists for IVF_FLAT and IVF_PQ"],
        "search_probes_device": [NOS, "probe-driven search only exists for IVF_FLAT and IVF_PQ"], "range_search": [13, 64],
        "range_search_nan": [0, 0], "shard_search": [18, 64], "shard_range_search": [17, 64],
        "shard_range_search_nan": [4, 0]},
    "ivf_flat_l2": {"search_64": [15, 64], "search_1": [4, 0], "search_device": [15, 64], "coarse_device": [2, 0],
        "search_probes_device": [13, 64], "range_search": [14, 64], "range_search_nan": [0, 0], "shard_search": [18, 64],
        "shard_range_search": [18, 64], "shard_range_search_nan": [6, 0]},
    "ivf_flat_cos": {"search_64": [16, 64], "search_1": [5, 0], "search_device": [16, 64], "coarse_device": [3, 0],
        "search_probes_device": [14, 64], "range_search": [15, 64], "range_search_nan": [0, 0], "shard_search": [19, 64],
        "shard_range_search": [19, 64], "shard_range_search_nan": [7, 0]},
    "ivf_pq8_l2": {"search_64": [5, 0], "search_1": [5, 0], "search_device": [5, 0], "coarse_device": [2, 0],
        "search_probes_device": [3, 0], "range_search": [5, 0], "range_search_nan": [0, 0], "shard_search": [8, 0],
        "shard_range_search": [9, 0], "shard_range_search_nan": [6, 0]},
    "ivf_pq4_ip": {"search_64": [5, 0], "search_1": [5, 0], "search_device": [5, 0], "coarse_device": [2, 0],
        "search_probes_device": [3, 0], "range_search": [5, 0], "range_search_nan": [0, 0], "shard_search": [8, 0],
        "shard_range_search": [9, 0], "shard_range_search_nan": [6, 0]},
    "ivf_pqflat_l2": {"search_64": [13, 64], "search_1": [15, 64], "search_device": [28, 64],
        "coarse_device": [NOS, "an IVF_PQ index in inner-Flat mode (too few training rows) has no inverted lists"],
        "search_probes_device": [NOS, "an IVF_PQ index in inner-Flat mode (too few training rows) has no inverted lists"],
        "range_search": [0, 0], "range_search_nan": [0, 0],
        "shard": [NOS, "an IVF_PQ index in inner-Flat mode (too few training rows) has no inverted lists to shard"]},
    "hnsw_l2": {"search_64": [1, 0], "search_1": [1, 0], "search_device": [1, 0],
        "coarse_device": [NOS, "coarse quantiser only exists for IVF_FLAT and IVF_PQ"],
        "search_probes_device": [NOS, "probe-driven search only exists for IVF_FLAT and IVF_PQ"],
        "range_search": [NOS, "RangeSearch not support in Hnsw!!!"], "shard_search": [4, 0],
        "shard_range_search": [NOS, "RangeSearch not support in Hnsw!!!"]},
    "hnsw_cos": {"search_64": [2, 0], "search_1": [2, 0], "search_device": [2, 0],
        "coarse_device": [NOS, "coarse quantiser only exists for IVF_FLAT and IVF_PQ"],
        "search_probes_device": [NOS, "probe-driven search only exists for IVF_FLAT and IVF_PQ"],
        "range_search": [NOS, "RangeSearch not support in Hnsw!!!"], "shard_search": [5, 0],
        "shard_range_search": [NOS, "RangeSearch not support in Hnsw!!!"]},
    "binary_flat": {"search_64": [3, 0], "search_1": [3, 0], "search_device": [3, 0],
        "coarse_device": [NOS, "coarse quantiser only exists for IVF_FLAT and IVF_PQ"],
        "search_probes_device": [NOS, "probe-driven search only exists for IVF_FLAT and IVF_PQ"], "range_search": [3, 0],
        "range_search_nan": [ILL, "radius is NaN"]},
    "binary_ivf": {"search_64": [5, 0], "search_1": [5, 0], "search_device": [5, 0],
        "coarse_device": [NOS, "coarse quantiser only exists for IVF_FLAT and IVF_PQ"],
        "search_probes_device": [NOS, "probe-driven search only exists for IVF_FLAT and IVF_PQ"], "range_search": [5, 0],
        "range_search_nan": [ILL, "radius is NaN"]},
}


@pytest.mark.parametrize("kind", KINDS)
def test_read_routes(kind):
    assert observe(kind) == EXPECTED[kind]
