"""Every sharded read entry point uses up its sequence number when it is refused (csrc/shard.cu, shard_read).

Batches are enqueued strictly in sequence order, so a refused read that left its number unused would make the next batch
wait for it forever.  For each read (top-k, deep and range; host and device pointers; the float and the _binary entry
points) at a world of one: a refused call at `seq`, then the same `seq` again is refused as already used, and the next
call at `seq + 1` answers."""
import ctypes

import numpy as np
import pytest

import b200vs
from b200vs import BINARY_FLAT, EILLEGAL_PARAMETERS, HAMMING, IVF_FLAT, L2
from gpu_util import require_gpu

pytestmark = pytest.mark.gpu
D, BDIM, NLIST, NQ, K = 16, 64, 16, 4, 5


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def _shard(binary):
    rng = np.random.default_rng(7)
    ids = np.arange(2000, dtype=np.int64)
    if binary:
        sh = b200vs.BinaryShard(b200vs.Index(BINARY_FLAT, HAMMING, BDIM), 0, 1, None)
        sh.add(rng.integers(0, 256, (2000, BDIM // 8), dtype=np.uint8), ids)
        return sh, rng.integers(0, 256, (NQ, BDIM // 8), dtype=np.uint8)
    ix = b200vs.Index(IVF_FLAT, L2, D, nlist=NLIST)
    ix.train(rng.standard_normal((3000, D)).astype(np.float32))
    ix.add(rng.standard_normal((2000, D)).astype(np.float32), ids)
    return b200vs.Shard(ix, 0, 1, None), rng.standard_normal((NQ, D)).astype(np.float32)


@pytest.mark.parametrize("binary", [False, True])
def test_refused_reads_use_their_sequence_number(binary):
    import torch
    sh, xq = _shard(binary)
    L = b200vs.lib()
    sp, _ = b200vs.make_search_params(nprobe=4)
    sp = ctypes.byref(sp)
    sfx = "_binary" if binary else ""
    od, oi, oc = np.zeros((NQ, K), np.float32), np.zeros((NQ, K), np.int64), np.zeros(NQ, np.int32)
    od_t = torch.zeros((NQ, K), dtype=torch.float32, device="cuda")
    oi_t = torch.zeros((NQ, K), dtype=torch.int64, device="cuda")
    oc_t = torch.zeros(NQ, dtype=torch.int32, device="cuda")
    xq_t = torch.from_numpy(xq).cuda()
    torch.cuda.synchronize()
    x, xd = xq.ctypes.data, xq_t.data_ptr()
    h, hd = (od.ctypes.data, oi.ctypes.data), (od_t.data_ptr(), oi_t.data_ptr())
    reads = {  # name: call(seq, nq)
        "search": lambda s, n: getattr(L, f"b200vs_shard_search{sfx}")(sh.h, s, n, x, K, sp, *h),
        "search_device": lambda s, n: getattr(L, f"b200vs_shard_search{sfx}_device")(sh.h, s, n, xd, K, sp, *hd, None),
        "search_deep": lambda s, n: getattr(L, f"b200vs_shard_search{sfx}_deep")(sh.h, s, n, x, K, sp, *h),
        "range_search": lambda s, n: getattr(L, f"b200vs_shard_range_search{sfx}")(sh.h, s, n, x, 1e9, K, sp, *h, oc.ctypes.data),
        "range_search_device": lambda s, n: getattr(L, f"b200vs_shard_range_search{sfx}_device")(
            sh.h, s, n, xd, 1e9, K, sp, *hd, oc_t.data_ptr(), None),
    }
    seq = 0
    for name, call in reads.items():
        assert call(seq, 0) == EILLEGAL_PARAMETERS, f"{name}: an empty batch was not refused"
        assert call(seq, NQ) == EILLEGAL_PARAMETERS and "sequence number already used" in L.b200vs_last_error().decode(), \
            f"{name}: the refused call left seq {seq} unused"
        oi[:] = -1
        oi_t.fill_(-1)
        torch.cuda.synchronize()
        rc = call(seq + 1, NQ)
        assert rc == b200vs.OK, f"{name}: the next batch failed: {L.b200vs_last_error().decode()}"
        torch.cuda.synchronize()
        got = oi_t.cpu().numpy() if name.endswith("_device") else oi
        assert (got >= 0).all(), f"{name}: the next batch returned no rows"
        seq += 2
    sh.close()
