"""sm_90a kernel numerics vs plain PyTorch fp32 references (runs on an H100: `pytest -m gpu`).
The checks themselves live in bench_tools/gpu_check.py so they can also be run stand-alone."""
import pytest

from bench_tools import gpu_check

pytestmark = pytest.mark.gpu


def test_native_library_is_loaded_not_a_fallback():
    from dist_mnist_b200 import _native as N
    lib = N.lib()
    assert lib is not None
    maps = open("/proc/self/maps").read()
    assert "libdmnist_sm90a.so" in maps


def test_wgmma_forward_gemm():
    assert gpu_check.check_gemm_fwd()


def test_wgmma_dw_gemm_with_push_epilogue():
    assert gpu_check.check_gemm_dw()


def test_wgmma_dx_gemm():
    assert gpu_check.check_gemm_dx()


def test_fused_softmax_ce_head():
    assert gpu_check.check_head()


def test_accuracy_reduction():
    assert gpu_check.check_accuracy()


def test_persistent_ps_serve_kernel():
    assert gpu_check.check_ps_serve()


def test_dense_apply_vs_torch_optim():
    assert gpu_check.check_dense_apply()


def test_p2p_copy_kernels_local():
    assert gpu_check.check_p2p_local()
