"""CPU: `plan_gemm` gives single-wave long-K GEMMs whose A reads dominate a 1 x 2 cluster that multicasts A, and leaves
every other plan on single CTAs."""
import ctypes


def _plan(m, n, k, epi):
    from pipeedge_b200 import _lib
    out = (ctypes.c_int * 6)()
    _lib.check(_lib.LIB.pe_debug_gemm_plan(m, n, k, epi, out))
    return dict(zip(('cm', 'cn', 'bn', 'stages', 'tiles', 'ctas'), out))


def test_vit_base_fc2_plans_a_pair_that_shares_a():
    from pipeedge_b200 import _lib
    for epi in (_lib.PE_EPI_F32, _lib.PE_EPI_RESID_F32):
        assert _plan(8 * 197, 768, 3072, epi) == {'cm': 1, 'cn': 2, 'bn': 96, 'stages': 7, 'tiles': 104, 'ctas': 104}


def test_other_long_k_plans_stay_single_cta():
    from pipeedge_b200 import _lib
    f32 = _lib.PE_EPI_F32
    vit_l = _plan(16 * 197, 1024, 4096, f32)          # 125 tiles of BN 224: pairs would need a second wave
    assert (vit_l['cm'], vit_l['cn'], vit_l['bn'], vit_l['tiles']) == (1, 1, 224, 125)
    bert = _plan(32 * 128, 768, 3072, f32)            # BN 192: halving A cuts a tile's bytes by only a fifth
    assert (bert['cm'], bert['cn'], bert['bn'], bert['tiles']) == (1, 1, 192, 128)
    for m, n, k in ((8 * 197, 2304, 768), (8 * 197, 768, 768), (8 * 197, 3072, 768), (4096, 3072, 768)):
        p = _plan(m, n, k, f32)
        assert (p['cm'], p['cn']) == (1, 1), (m, n, k, p)
