"""-m gpu: the weight packer of the tensor-core kernels (tc_pack) writes the bf16 split-plane image that the wgmma B operand and the
1-D bulk-copy weight ring expect, [K-block of 32][plane][k/8][row][8 bf16], rows padded to whole n64 blocks with zeros."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("K,N,planes", [(32, 16, 1), (64, 80, 2), (96, 256, 2), (256, 96, 1), (128, 200, 2)])
def test_tc_pack_layout(K, N, planes):
    import sdfstudio_b200 as sb

    lib = sb._lib.load_debug()
    g = torch.Generator().manual_seed(K * 7 + N)
    A = torch.randn(128, K, generator=g).cuda()
    W = torch.randn(N, K, generator=g).cuda()
    Np = (N + 15) // 16 * 16
    Np64 = (N + 63) // 64 * 64
    D = torch.empty(128, Np, device="cuda")
    scratch = torch.full(((K // 32) * planes * Np64 * 64,), 0x7F, dtype=torch.uint8, device="cuda")   # not a valid packed image
    rc = lib.sdfb200_debug_tc_gemm(A.data_ptr(), W.data_ptr(), K, N, 0, planes, D.data_ptr(), scratch.data_ptr(), 0)
    assert rc == 0, lib.sdfb200_last_error_string()
    torch.cuda.synchronize()

    hi = W.bfloat16()
    lo = (W - hi.float()).bfloat16()
    want = torch.zeros(K // 32, planes, 4, Np64, 8, dtype=torch.bfloat16, device="cuda")
    for p, part in enumerate((hi, lo)[:planes]):
        # element (n, k) -> [k / 32][p][(k % 32) / 8][n][k % 8]
        want[:, p, :, :N, :] = part.view(N, K // 32, 4, 8).permute(1, 2, 0, 3)
    got = scratch.view(torch.bfloat16).view(K // 32, planes, 4, Np64, 8)
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))
