"""The fixed-order cross-CTA reduction (common.cuh launch_ordered_sum): out[i] += part[0][i] + part[1][i] + ... added strictly in
part order, so the result must equal, bit for bit, the same additions done one part at a time -- for few parts (one thread per
element) and for many (parts staged through shared memory), float32 and float64."""
import pytest
import torch

import rlr_b200  # noqa: F401
from rlr_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.mark.parametrize("nparts,n,dtype", [
    (264, 256, torch.float32), (396, 2048, torch.float32), (65, 33, torch.float32), (16, 100, torch.float32),
    (300, 1, torch.float32), (132, 1, torch.float64), (15, 4096, torch.float32), (2, 5000, torch.float32),
])
def test_ordered_sum_adds_in_part_order(nparts, n, dtype):
    torch.manual_seed(nparts + n)
    # magnitudes spread over several decades so that any other association order changes the rounding
    part = (torch.randn(nparts, n, device=DEV, dtype=torch.float64) * torch.logspace(-3, 3, nparts, device=DEV,
                                                                                    dtype=torch.float64)[:, None]).to(dtype)
    out = torch.randn(n, device=DEV, dtype=dtype)
    s = part[0].clone()
    for j in range(1, nparts):
        s = s + part[j]
    want = out + s
    ops.ext().ordered_sum(out, part)
    torch.cuda.synchronize()
    assert torch.equal(out, want)
