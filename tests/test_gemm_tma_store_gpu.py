"""GPU: the GEMM's TMA-store epilogue gives the bits of the register-store epilogue and writes nothing outside `out`.

Every epilogue that stores through TMA (F16, GELU_F16, F32, RESID_F32, TANH_F32) runs at M in {1, 40, 127, 128, 1576},
with N ragged against the tile width, on one-round and multi-round plans, a 1 x 2 multicast cluster, BN 256 (fp32 tiles
that leave in two passes) and the planner's own choice. The library reads PE_GEMM_REG_STORE once per process, so two
child processes run the same cases, one per store path, and the outputs must be `torch.equal`. Each output sits inside
a NaN guard band (more than a whole tile wide on both sides) that must come back untouched, and no NaN may remain in
the output itself.
"""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPILOGUES = ['PE_EPI_F16', 'PE_EPI_GELU_F16', 'PE_EPI_F32', 'PE_EPI_RESID_F32', 'PE_EPI_TANH_F32']
ROWS = [1, 40, 127, 128, 1576]
# (n, k, forced plan "CM,CN,BN" or None): every n is ragged against its BN except the planner's own 768
PLANS = [
    (200, 256, '1,1,64'),      # one round
    (4360, 128, '1,1,32'),     # 137 column tiles: two or more rounds at every M
    (520, 192, '1,1,256'),     # fp32 tiles go out in two passes of four boxes
    (776, 3072, '1,2,96'),     # 1 x 2 cluster, A multicast, long K
    (768, 768, None),          # the planner's plan (ViT-B out-proj shape)
]

_CHILD = """
import os, sys
sys.path[:0] = [sys.argv[1], os.path.join(sys.argv[1], 'tests')]
import test_gemm_tma_store_gpu as T
sys.exit(T.child_main(sys.argv[2]))
"""


def _case_id(epi_name, m, n, k, force):
    return f"{epi_name}-m{m}-n{n}-k{k}-{force or 'auto'}"


def child_main(dest):
    """Runs every case on this process's store path; saves the outputs to `dest`, prints guard-band failures."""
    from pipeedge_b200 import _lib, ops
    dev = torch.device('cuda', 0)
    outs, failures = {}, []
    for n, k, force in PLANS:
        if force is None:
            os.environ.pop('PE_GEMM_FORCE', None)
        else:
            os.environ['PE_GEMM_FORCE'] = force
        gen = torch.Generator(device=dev).manual_seed(n * 31 + k)
        a_all = torch.randn(max(ROWS), k, device=dev, generator=gen).half()
        w = (torch.randn(n, k, device=dev, generator=gen) * 0.05).half()
        bias = torch.randn(n, device=dev, generator=gen)
        resid_all = torch.randn(max(ROWS), n, device=dev, generator=gen)
        for m in ROWS:
            for epi_name in EPILOGUES:
                epi = getattr(_lib, epi_name)
                dtype = torch.float16 if 'F16' in epi_name else torch.float32
                guard = 130 * n                       # > one 128-row tile; a multiple of 8 keeps `out` 16-byte aligned
                buf = torch.full((guard + m * n + guard,), float('nan'), dtype=dtype, device=dev)
                out = buf[guard:guard + m * n].view(m, n)
                resid = resid_all[:m].contiguous() if epi_name == 'PE_EPI_RESID_F32' else None
                ops.linear(a_all[:m].contiguous(), w, bias, epi, resid=resid, out=out)
                torch.cuda.synchronize()
                cid = _case_id(epi_name, m, n, k, force)
                if not (torch.isnan(buf[:guard]).all() and torch.isnan(buf[guard + m * n:]).all()):
                    failures.append(f"{cid}: wrote outside out")
                if torch.isnan(out).any():
                    failures.append(f"{cid}: left {int(torch.isnan(out).sum())} elements of out unwritten")
                outs[cid] = out.cpu()
    os.environ.pop('PE_GEMM_FORCE', None)
    torch.save(outs, dest)
    print('\n'.join(failures) if failures else 'all ok', flush=True)
    return 1 if failures else 0


def _run_child(dest, reg_store):
    env = {k: v for k, v in os.environ.items() if k not in ('PE_GEMM_REG_STORE', 'PE_GEMM_FORCE')}
    if reg_store:
        env['PE_GEMM_REG_STORE'] = '1'
    res = subprocess.run([sys.executable, '-c', _CHILD, ROOT, dest], capture_output=True, text=True, timeout=1800,
                         env=env)
    assert res.returncode == 0 and 'all ok' in res.stdout, res.stdout[-6000:] + res.stderr[-4000:]
    return torch.load(dest)


@pytest.fixture(scope='module')
def both_paths(tmp_path_factory):
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    d = tmp_path_factory.mktemp('gemm_store')
    return _run_child(str(d / 'tma.pt'), False), _run_child(str(d / 'reg.pt'), True)


@pytest.mark.parametrize('epi_name', EPILOGUES)
def test_tma_store_equals_register_store(both_paths, epi_name):
    tma, reg = both_paths
    ids = [_case_id(epi_name, m, n, k, force) for n, k, force in PLANS for m in ROWS]
    bad = [cid for cid in ids if not torch.equal(tma[cid], reg[cid])]
    assert not bad, f"TMA-stored output differs from the register-stored one: {bad}"
