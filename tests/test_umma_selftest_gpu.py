"""Pins the wgmma shared-memory descriptor encoding on real hardware: one 128xNxK (and 64xNxK,
and MN-major) MMA through hrf_selftest_umma against torch.  If the expected (LBO,SBO) reading is
wrong, the failing assert prints which alternative matches."""
import pytest
import torch

from humanrf_b200 import _lib as L

pytestmark = pytest.mark.gpu


def run(cuda, m, n, k, mn_major, a_k, a_m, b_k, b_n, a_lbo, a_sbo, b_lbo, b_sbo, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    a = torch.randn(m, k, generator=g).to(torch.bfloat16).to(cuda)
    b = torch.randn(n, k, generator=g).to(torch.bfloat16).to(cuda)
    d = torch.full((m, n), float("nan"), device=cuda)
    L.check(L.lib().hrf_selftest_umma(a.data_ptr(), b.data_ptr(), d.data_ptr(), m, n, k, a_k, a_m, b_k, b_n, a_lbo,
                                      a_sbo, b_lbo, b_sbo, mn_major, L.stream()))
    torch.cuda.synchronize()
    ref = a.float() @ b.float().t()
    return (d - ref).abs().max().item()


@pytest.mark.parametrize("n,k", [(64, 32), (16, 64), (64, 64), (32, 64)])
def test_k_major_m128(cuda, n, k):
    # operand tiles exactly as the field kernels lay them out (csrc/field_common.cuh)
    a_k, a_m = 2048, 128
    b_k, b_n = (n // 8) * 128, 128
    err = run(cuda, 128, n, k, 0, a_k, a_m, b_k, b_n, a_k, a_m, b_k, b_n)
    if not err < 1e-2:
        alt = run(cuda, 128, n, k, 0, a_k, a_m, b_k, b_n, a_m, a_k, b_n, b_k)
        pytest.fail(f"K-major LBO=k-stride/SBO=m-stride gives err {err}; swapped gives {alt}")


@pytest.mark.parametrize("m,n", [(64, 32), (64, 64), (64, 16), (128, 64), (128, 32)])
def test_mn_major(cuda, m, n):
    # wgrad / dgrad view: contraction over k with the MN dimension contiguous
    k = 128 if m == 64 else 64
    a_k, a_m = 128, 2048
    b_k, b_n = 128, 2048
    err = run(cuda, m, n, k, 3, a_k, a_m, b_k, b_n, a_k, a_m, b_k, b_n)
    if not err < 2e-2:
        alt = run(cuda, m, n, k, 3, a_k, a_m, b_k, b_n, a_m, a_k, b_n, b_k)
        pytest.fail(f"MN-major LBO=k-stride/SBO=mn-stride gives err {err}; swapped gives {alt}")


@pytest.mark.parametrize("n_in,k_out", [(64, 16), (64, 64), (32, 64)])
def test_dgrad_mixed_major(cuda, n_in, k_out):
    # dgrad: A = gradient tile (K-major), B = forward weight blob W[k_out, n_in] read MN-major:
    # B(n'=in, k'=out) lives at (in/8)*(k_out/8)*128 + (out/8)*128 + (out%8)*16 + (in%8)*2
    a_k, a_m = 2048, 128
    b_k, b_n = 128, (k_out // 8) * 128
    err = run(cuda, 128, n_in, k_out, 2, a_k, a_m, b_k, b_n, a_k, a_m, b_k, b_n)
    assert err < 2e-2, err
