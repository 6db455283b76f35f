"""GPU tests of the tensor-core GEMM's tile plan: 256- and 128-row output tiles on both tensor-core backends against an fp64
reference (bounds of test_gpu_gemm.py: 1e-5 of max |C|, 2e-5 with accumulation).  Every case first asserts, through
ase_gemm_tc_plan, which tile the shape runs on, so a change of the plan cannot silently move a case to the other tile.

Tile shapes (rows x cols, ring stages): 256 x 128 (2), 256 x 64 (2), 128 x 128 (3), 128 x 64 (4).  A k-block is 64 halfs
(backend 2) or 32 TF32 words (backend 1); each consumer warpgroup owns half of the tile's rows as one or two m64 blocks."""
import pytest
import torch

pytestmark = pytest.mark.gpu

TC_BACKENDS = [1, 2]
MAJORS = [(False, False), (False, True), (True, False), (True, True)]


def _plan(M, N, K, tc, accumulate=False, split_k=0):
    from ase_b200 import ops
    return ops.gemm_tc_plan(M, N, K, accumulate, split_k, tc)


def _run(M, N, K, a_trans, b_trans, tc, tile, bias=False, act=0, mask_mode=0, mask_bits=False, accumulate=False, split_k=0,
         alpha=1.0, colsum=False, relu_bits=False, splits=None, lda_pad=0, tol=None, seed=0):
    """C = epi(alpha op(A) op(B)) through ase_gemm against fp64; tile = (rows, cols) the plan must pick."""
    from ase_b200 import ops
    plan = _plan(M, N, K, tc, accumulate, split_k)
    assert plan[:2] == tile, ((M, N, K, accumulate, split_k, tc), plan, tile)
    if splits is not None:
        assert plan[2] == splits, ((M, N, K, split_k, tc), plan)
    g = torch.Generator().manual_seed(seed + M + 7 * N + 13 * K)
    A = torch.randn((K, M + lda_pad) if a_trans else (M, K + lda_pad), generator=g).cuda()
    B = torch.randn((K, N + lda_pad) if b_trans else (N, K + lda_pad), generator=g).cuda()
    Av = A[:, :M] if a_trans else A[:, :K]
    Bv = B[:, :N] if b_trans else B[:, :K]
    bias_t = torch.randn(N, generator=g).cuda() if bias else None
    mask_src = torch.randn(M, N, generator=g).cuda().clamp(-0.9, 0.9) if mask_mode else None
    bits_in = None
    if mask_bits:
        assert mask_mode == 1
        cols = torch.arange(N, device='cuda')
        pos = (mask_src > 0).int() << (cols % 32).int()
        bits_in = torch.zeros(M, (N + 31) // 32, dtype=torch.int64, device='cuda').index_add_(1, (cols // 32), pos.long())
        bits_in = ((bits_in + 2 ** 31) % 2 ** 32 - 2 ** 31).int()
    out, base = None, 0
    if accumulate:
        out = torch.randn(M, N, generator=g).cuda()
        base = out.double().clone()
    cs = torch.zeros(N, device='cuda') if colsum else None
    rb = torch.zeros(M, (N + 31) // 32, dtype=torch.int32, device='cuda') if relu_bits else None
    C = ops.gemm(Av, Bv, a_trans, b_trans, bias_t, act, mask_src, mask_mode, out, accumulate, split_k, alpha, tc,
                 colsum_out=cs, relu_bits_out=rb, mask_bits=bits_in)
    torch.cuda.synchronize()
    a = Av.double().t() if a_trans else Av.double()
    b = Bv.double() if b_trans else Bv.double().t()
    ref = alpha * (a @ b)
    if bias_t is not None:
        ref = ref + bias_t.double()
    if act == 1:
        ref = torch.relu(ref)
    elif act == 2:
        ref = torch.tanh(ref)
    if mask_mode == 1:
        ref = ref * (mask_src > 0).double()
    elif mask_mode == 2:
        ref = ref * (1 - mask_src.double() ** 2)
    full = ref + base
    tol = tol or (2e-5 if accumulate else 1e-5)
    err = float((C.double() - full).abs().max() / full.abs().max())
    assert err < tol, ((M, N, K, a_trans, b_trans, tc, plan), err)
    if colsum:
        s = ref.sum(0)
        assert float((cs.double() - s).abs().max() / s.abs().max()) < 2e-5, (M, N, K, tc)
    if relu_bits:
        cols = torch.arange(N, device='cuda')
        assert torch.equal(((rb[:, cols // 32] >> (cols % 32)) & 1).bool(), C > 0), (M, N, K, tc)
        if N % 32:
            assert int((rb[:, -1].long() & 0xFFFFFFFF >> (N % 32) << (N % 32)).abs().max()) == 0
    return C


def test_plan_picks_tiles():
    """The plan's choices the other tests rely on, and the learner's shapes that must stay at 128 rows."""
    for tc in TC_BACKENDS:
        assert _plan(32768, 1024, 1024, tc) == (256, 128, 1)         # actor forward / dX: 512 CTAs instead of 1024
        assert _plan(32768, 64, 256, tc) == (256, 64, 1)
        assert _plan(4096, 512, 1024, tc) == (128, 128, 1)           # Ba x 512: 64 CTAs at 256 rows would leave half the SMs idle
        assert _plan(12288, 512, 1024, tc) == (128, 128, 1)
        assert _plan(300, 1, 512, tc) == (128, 64, 1)                # value / logit heads
        assert _plan(1024, 1024, 32768, tc, True, 9) == (128, 128, 9)    # an explicit split count is kept
        assert _plan(1024, 1024, 32768, tc, True, 0)[2] == 1             # 0 = no split
        assert _plan(1024, 1024, 32768, tc, False, 9)[2] == 1            # no split-K without accumulate
        bm, bn, s = _plan(1024, 1024, 32768, tc, True, -1)               # the learner's dW: the plan picks the splits
        assert 1 < s <= 16 and _plan(1024, 1024, 32768, tc, True, s) == (bm, bn, s)


@pytest.mark.parametrize('tc', TC_BACKENDS)
@pytest.mark.parametrize('a_trans,b_trans', MAJORS)
def test_tall_tiles_ragged(a_trans, b_trans, tc):
    """256-row tiles: M tails inside the last tile (the second warpgroup without valid rows, the second m64 block of the first
    warpgroup without valid rows, both warpgroups partly valid), an N tail, K not a multiple of the k-block, unaligned ld."""
    _run(16448, 1000, 317, a_trans, b_trans, tc, (256, 128))                    # last tile: 64 valid rows (warpgroup 1 idle)
    _run(16576, 1000, 317, a_trans, b_trans, tc, (256, 128), lda_pad=3)         # last tile: 192 valid rows
    _run(8320, 1024, 31, a_trans, b_trans, tc, (256, 128))                      # 128 valid rows, K = 31: one partial k-block
    _run(8192, 1024, 1, a_trans, b_trans, tc, (256, 128))                       # K = 1 outer product
    _run(32768, 50, 317, a_trans, b_trans, tc, (256, 64))                       # 256 x 64 tiles, N tail


@pytest.mark.parametrize('tc', TC_BACKENDS)
@pytest.mark.parametrize('a_trans,b_trans', MAJORS)
def test_short_tiles_ragged(a_trans, b_trans, tc):
    """128-row tiles chosen by the plan for shapes with too few 256-row tiles to fill the SMs."""
    _run(4096, 500, 317, a_trans, b_trans, tc, (128, 128), lda_pad=3)
    _run(4096, 64, 31, a_trans, b_trans, tc, (128, 64))
    _run(200, 40, 50, a_trans, b_trans, tc, (128, 64))
    _run(300, 1, 512, a_trans, b_trans, tc, (128, 64))


@pytest.mark.parametrize('tc', TC_BACKENDS)
def test_ring_wrap_every_stage_count(tc):
    """More k-blocks than ring stages on all four tile shapes (2, 2, 3 and 4 stages): every stage is refilled several times and
    both barrier parities are used, with odd and even k-block counts."""
    _run(8192, 1024, 1024, False, False, tc, (256, 128), bias=True, act=1)       # 256 x 128, 2 stages
    _run(8192, 1024, 1040, False, True, tc, (256, 128))                           # an odd number of k-blocks
    _run(32768, 64, 1024, True, False, tc, (256, 64))                             # 256 x 64, 2 stages
    _run(4096, 512, 1024, False, True, tc, (128, 128), mask_mode=1)               # 128 x 128, 3 stages
    _run(4096, 64, 1040, True, True, tc, (128, 64))                               # 128 x 64, 4 stages


@pytest.mark.parametrize('tc', TC_BACKENDS)
def test_tall_tile_epilogues(tc):
    """The store phase of 256-row tiles, fast path (interior tiles, BN = 128) and generic path (tails, BN = 64, accumulate)."""
    _run(8192, 1024, 192, False, False, tc, (256, 128), bias=True, act=1, relu_bits=True)
    _run(8320, 1000, 192, False, False, tc, (256, 128), bias=True, act=1, relu_bits=True)      # M and N tails
    _run(8192, 1024, 256, False, False, tc, (256, 128), bias=True, act=2, alpha=1.0 / 16, tol=3e-5)   # O(1) pre-activations
    _run(8192, 1024, 512, False, True, tc, (256, 128), mask_mode=1, colsum=True)               # fp32 mask + column sums
    _run(8320, 1000, 512, False, True, tc, (256, 128), mask_mode=1, mask_bits=True, colsum=True)   # bit mask, tails
    _run(8192, 1024, 256, False, True, tc, (256, 128), mask_mode=2)
    _run(32768, 64, 256, False, False, tc, (256, 64), bias=True, act=2, alpha=1.0 / 16, tol=3e-5)
    _run(32768, 50, 256, False, True, tc, (256, 64), mask_mode=1, mask_bits=True, colsum=True)


@pytest.mark.parametrize('tc', TC_BACKENDS)
def test_tall_tile_split_k(tc):
    """Split-K with 256-row tiles: fp32 RED into C, a short last split, the learner's own choice of splits."""
    _run(1024, 1400, 12300, True, True, tc, (256, 128), accumulate=True, split_k=3, splits=3)     # last split one k-block short
    _run(2048, 1024, 4096, True, True, tc, (256, 128), accumulate=True, split_k=2, splits=2)
    s = _plan(1024, 1400, 4096, tc, True, -1)[2]
    _run(1024, 1400, 4096, True, True, tc, (256, 128), accumulate=True, split_k=s, splits=s)
    _run(8320, 1000, 317, False, False, tc, (256, 128), accumulate=True)                       # accumulate without split
    _run(1100, 1400, 12300, True, True, tc, (128, 128), accumulate=True, split_k=3, splits=3)
