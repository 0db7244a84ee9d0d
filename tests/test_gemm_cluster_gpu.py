"""GPU: a GEMM the planner gives a multicast cluster computes bit for bit what the same tiles compute as single CTAs:
a clustered tile runs the same wgmmas over the same K order on the same bytes; only the data movement differs."""
import ctypes
import pytest
import torch

pytestmark = pytest.mark.gpu


def _plan(m, n, k, epi):
    from pipeedge_b200 import _lib
    out = (ctypes.c_int * 6)()
    _lib.check(_lib.LIB.pe_debug_gemm_plan(m, n, k, epi, out))
    return dict(zip(('cm', 'cn', 'bn'), out[:3]))


@pytest.mark.parametrize('m, n, k', [(8 * 197, 768, 3072), (4 * 197, 768, 3072), (1000, 704, 2048)])
@pytest.mark.parametrize('epi_name', ['PE_EPI_F32', 'PE_EPI_RESID_F32'])
def test_clustered_plan_equals_single_cta_plan(m, n, k, epi_name, monkeypatch):
    from pipeedge_b200 import _lib, ops
    epi = getattr(_lib, epi_name)
    plan = _plan(m, n, k, epi)
    assert plan['cm'] * plan['cn'] > 1, plan
    gen = torch.Generator(device='cuda').manual_seed(m + n + k)
    a = torch.randn(m, k, device='cuda', generator=gen).half()
    w = (torch.randn(n, k, device='cuda', generator=gen) * 0.05).half()
    bias = torch.randn(n, device='cuda', generator=gen)
    resid = torch.randn(m, n, device='cuda', generator=gen) if epi == _lib.PE_EPI_RESID_F32 else None
    got = ops.linear(a, w, bias, epi, resid=resid)
    monkeypatch.setenv('PE_GEMM_FORCE', f"1,1,{plan['bn']}")
    want = ops.linear(a, w, bias, epi, resid=resid)
    torch.cuda.synchronize()
    assert torch.equal(got, want)
