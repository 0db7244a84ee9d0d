"""GPU: the wgmma attention kernel writes its context through one TMA store per (64 query rows, head, item), clipped by
a 3-D tensor map at each item's S. For every S it handles, on several batch and head counts: every context row is
written, nothing around the context is, and each item's rows are bit for bit what the kernel computes for that item
alone - the clip at the item boundary neither drops a row nor lets a tile spill into the next item."""
import pytest
import torch

pytestmark = pytest.mark.gpu

GUARD = 64   # rows of NaN before and after the context


def _attention(qkv, batch, tokens, heads):
    from pipeedge_b200._lib import LIB, check
    width = heads * 64
    buf = torch.full(((batch * tokens) + 2 * GUARD, width), float('nan'), dtype=torch.float16, device='cuda')
    ctx = buf[GUARD:GUARD + batch * tokens]
    check(LIB.pe_attention(qkv.data_ptr(), ctx.data_ptr(), batch, tokens, heads, 64,
                           torch.cuda.current_stream().cuda_stream))
    return buf


@pytest.mark.parametrize('batch, heads', [(1, 1), (3, 2), (2, 5)])
def test_context_rows_written_once_per_item(batch, heads):
    for tokens in range(1, 257):
        gen = torch.Generator(device='cuda').manual_seed(tokens)
        qkv = torch.randn(batch * tokens, 3 * heads * 64, device='cuda', generator=gen).half()
        buf = _attention(qkv, batch, tokens, heads)
        alone = [_attention(qkv[b * tokens:(b + 1) * tokens].clone(), 1, tokens, heads) for b in range(batch)]
        torch.cuda.synchronize()
        where = f'B={batch} S={tokens} H={heads}'
        assert torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[-GUARD:]).all(), f'{where}: wrote outside ctx'
        ctx = buf[GUARD:-GUARD]
        assert not torch.isnan(ctx).any(), f'{where}: context rows left unwritten'
        for b in range(batch):
            assert torch.equal(ctx[b * tokens:(b + 1) * tokens], alone[b][GUARD:-GUARD]), f'{where}: item {b} differs'
