"""The CUDA k-way merge (b200vs_merge_topk_device) follows the same rule as b200vs.shard.merge_topk."""
import numpy as np
import pytest

import b200vs
from b200vs import shard
from gpu_util import require_gpu

pytestmark = pytest.mark.gpu


def _parts(rng, nparts, nq, k, kind):
    pd = np.sort(rng.random((nparts, nq, k)).astype(np.float32), axis=2)
    pd[:, :, :2] = np.round(pd[:, :, :2], 1)  # force some ties
    pi = rng.permutation(nparts * nq * k).reshape(nparts, nq, k).astype(np.int64)
    pi[0, 0, k - 1] = -1
    if kind == "dead_part":  # one part holds no result at all
        pi[1] = -1
        pd[1] = 0
    elif kind == "holes":  # -1 entries in the middle of a part
        pi[:, :, 1:k - 1:3] = -1
    elif kind == "negative":
        pd = pd - np.float32(0.5)
        pd[:, :, :3] = np.float32(-0.25)
    elif kind == "signed_zero":  # -0.0 and +0.0 compare equal: the id decides
        pd[:, :, :4] = 0.0
        pd[::2, :, :2] = -0.0
    return np.sort(pd, axis=2, kind="stable"), pi


CASES = [  # (nparts, nq, k, kind)
    (2, 7, 5, "ties"), (8, 64, 10, "ties"), (4, 3, 100, "ties"),
    (8, 3, 4096, "ties"),       # 32768 candidates through an 8192-entry pool: it prunes
    (1, 5, 10, "ties"),
    (3, 4, 50, "dead_part"), (3, 4, 50, "holes"), (4, 6, 40, "negative"), (4, 6, 40, "signed_zero"),
]


def test_merge_kernel_matches_numpy_rule():
    require_gpu()
    import torch
    rng = np.random.default_rng(0)
    for nparts, nq, k, kind in CASES:
        case = f"nparts={nparts} nq={nq} k={k} {kind}"
        pd, pi = _parts(rng, nparts, nq, k, kind)
        td, ti = torch.from_numpy(pd).cuda(), torch.from_numpy(pi).cuda()
        od = torch.empty((nq, k), dtype=torch.float32, device="cuda")
        oi = torch.empty((nq, k), dtype=torch.int64, device="cuda")
        b200vs.merge_topk_device(0, nparts, nq, k, td.data_ptr(), ti.data_ptr(), od.data_ptr(), oi.data_ptr(), torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        wd, wi = shard.merge_topk(pd, pi, k)
        gd = od.cpu().numpy()
        assert np.array_equal(oi.cpu().numpy(), wi), case
        assert np.array_equal(gd, wd), case
        # bit for bit, except that the kernel's keys fold -0.0 into +0.0
        assert np.array_equal(gd.view(np.uint32), np.where(wd == 0, np.float32(0), wd).view(np.uint32)), case
        if kind == "signed_zero":
            assert (pd == 0).sum() > 0 and np.signbit(pd[pd == 0]).any(), "premise: -0.0 among the inputs"
