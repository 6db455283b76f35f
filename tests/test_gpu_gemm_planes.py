"""GPU tests of the operand-plane registry the learner runs every tensor-core GEMM through (PlaneRegistry, csrc/gemm_tc.cu), one GEMM
at a time, through the ase_gemm_planes_* handle of the C ABI.  ase_gemm (test_gpu_gemm*.py) never reaches the registry: only here
are the planes an epilogue writes, the elided fp32 store (c_planes_only), predicted scales, cached MN-major planes, sub-view
operands and the output-plane rules checked element by element.

Two oracles:
  * bit level: the planes an epilogue writes are exactly the split of the fp32 C the same GEMM stored.  Backend 2: hi = half(C s),
    lo = half(C s - hi) (round to nearest even) at the predicted scale s, the power of two that puts the previous call's max |C|
    into [2^8, 2^9).  Backend 1: the TF32 split (round to nearest, ties away), no scale.
  * fp64 per GEMM: every output against fp64 of the operands it consumed -- the stored fp32 tensor, or (hi + lo) / s for a tensor
    whose fp32 store was elided -- at the bars of test_gpu_gemm.py: 1e-5 of max |C|, 2e-5 with accumulation / split-K.

A scenario runs its GEMM sequence over 4 calls: call 0 calibrates the scales exactly, calls 1 and 2 run on predicted scales (the
epilogues write the planes), and the sites are forgotten before call 3 (new parameters: exact again)."""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

TC_BACKENDS = [1, 2]
TOP_SITE = 9                  # predicted scales put the previous max into [2^(TOP_SITE-1), 2^TOP_SITE)
ERR_INVALID, ERR_WORKSPACE = -1, -3
SITES = 1024
WS_BYTES = 64 << 20
NAN = float('nan')


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return None if t is None else t.data_ptr()


def _site_scale(amax):
    """scale_from_amax(amax, TOP_SITE) of tc_common.cuh: 1 for an all-zero tensor."""
    amax = float(amax)
    if not (0.0 < amax < 3.0e38):
        return 1.0
    return math.ldexp(1.0, max(-100, min(100, TOP_SITE - math.frexp(amax)[1])))


def _split_f16(x, s):
    xs = x.float() * s                              # exact: s is a power of two
    hi = xs.half()
    return hi, (xs - hi.float()).half()


def _rna_tf32(x):
    """cvt.rna.tf32.f32: round to 10 mantissa bits, ties away from zero (finite inputs)."""
    b = (x.contiguous().view(torch.int32).long() & 0xFFFFFFFF) + 0x1000
    b = b & 0xFFFFE000
    return ((b + 2 ** 31) % 2 ** 32 - 2 ** 31).int().view(torch.float32)


def _split_tf32(x):
    hi = _rna_tf32(x)
    return hi, _rna_tf32(x - hi)


def _assert_bits_equal(got, want, what):
    it = torch.int16 if got.dtype == torch.float16 else torch.int32
    bad = (got.contiguous().view(it) != want.contiguous().view(it)).nonzero()
    if bad.numel():
        r, c = bad[0].tolist()
        raise AssertionError(f"{what}: {bad.shape[0]} elements differ, first at row {r} col {c}: "
                             f"got {float(got[r, c])!r}, want {float(want[r, c])!r}")


def _close(got, ref, tol, what):
    err = float((got.double() - ref).abs().max()) / max(float(ref.abs().max()), 1e-30)
    assert err < tol, (what, err)


def _mm(A, B, a_trans=False, b_trans=False):
    a = A.double().t() if a_trans else A.double()
    b = B.double() if b_trans else B.double().t()
    return a @ b


def _unpack_bits(bits, N):
    cols = torch.arange(N, device=bits.device)
    return ((bits[:, cols // 32] >> (cols % 32)) & 1).bool()


def _pack_bits(mask):
    M, N = mask.shape
    cols = torch.arange(N, device=mask.device)
    words = torch.zeros(M, (N + 31) // 32, dtype=torch.int64, device=mask.device)
    words.index_add_(1, cols // 32, mask.long() << (cols % 32))
    return ((words + 2 ** 31) % 2 ** 32 - 2 ** 31).int()


class Planes:
    """One PlaneRegistry behind the ase_gemm_planes_* handle, with its registered buffers, their planes and a GEMM workspace."""

    def __init__(self, backend):
        from ase_b200 import lib as L
        self.L, self.lib, self.backend = L, L.lib, backend
        self.dev = torch.zeros(self.lib.ase_gemm_planes_device_bytes(), dtype=torch.uint8, device='cuda') if backend == 2 else None
        h = C.c_void_p()
        L.check(self.lib.ase_gemm_planes_create(backend, _p(self.dev), C.byref(h)), 'ase_gemm_planes_create')
        self.h = h
        ws = torch.empty(WS_BYTES + 1024, dtype=torch.uint8, device='cuda')
        off = (-ws.data_ptr()) % 1024
        self.ws = ws[off:off + WS_BYTES]
        self.planes = {}
        self.scale_buf = torch.zeros(2, device='cuda')

    def close(self):
        torch.cuda.synchronize()
        self.lib.ase_gemm_planes_destroy(self.h)

    def buffer(self, rows, cols, init=None):
        """A registered fp32 buffer [rows, cols] with the learner's plane capacity (rows x cols padded to 4 fp32 words each)."""
        t = torch.zeros(rows, cols, device='cuda') if init is None else init.float().cuda().contiguous()
        cap = rows * ((cols + 3) // 4 * 4)
        hi, lo = torch.zeros(cap, device='cuda'), torch.zeros(cap, device='cuda')
        self.L.check(self.lib.ase_gemm_planes_add(self.h, t.data_ptr(), t.numel(), hi.data_ptr(), lo.data_ptr(), cap), 'ase_gemm_planes_add')
        self.planes[t.data_ptr()] = (hi, lo)
        return t

    def begin(self, base=0):
        self.L.check(self.lib.ase_gemm_planes_begin_call(self.h, base, _stream()), 'ase_gemm_planes_begin_call')

    def forget(self):
        self.L.check(self.lib.ase_gemm_planes_forget(self.h), 'ase_gemm_planes_forget')

    def prep_weights(self, ws):
        n = len(ws)
        src = (C.c_void_p * n)(*[w.data_ptr() for w in ws])
        rows = (C.c_int * n)(*[w.shape[0] for w in ws])
        cols = (C.c_int * n)(*[w.shape[1] for w in ws])
        self.L.check(self.lib.ase_gemm_planes_prep_weights(self.h, src, rows, cols, n, _stream()), 'ase_gemm_planes_prep_weights')

    def gemm(self, A, B, Cout, a_trans=False, b_trans=False, bias=None, act=0, mask_src=None, mask_mode=0, mask_bits=None,
             accumulate=False, split_k=0, alpha=1.0, planes_only=False, colsum=None, relu_bits=None):
        """C = epi(alpha op(A) op(B)) through the registry; A, B, C may be views (leading dimension = stride(0)).  Returns the status."""
        M, K = (A.shape[1], A.shape[0]) if a_trans else (A.shape[0], A.shape[1])
        N = B.shape[1] if b_trans else B.shape[0]
        assert (B.shape[0] if b_trans else B.shape[1]) == K and tuple(Cout.shape) == (M, N)
        assert A.stride(1) == 1 and B.stride(1) == 1 and Cout.stride(1) == 1
        assert self.lib.ase_gemm_tc_workspace_bytes(M, N, K) <= WS_BYTES
        p = self.L.GemmParams(_p(A), A.stride(0), int(a_trans), _p(B), B.stride(0), int(b_trans), _p(Cout), Cout.stride(0), M, N, K, alpha,
                              _p(bias), act, _p(mask_src), 0 if mask_src is None else mask_src.stride(0), mask_mode, int(accumulate),
                              split_k, self.backend, _p(self.ws), WS_BYTES, _p(colsum), _p(relu_bits),
                              0 if relu_bits is None else relu_bits.stride(0), _p(mask_bits), 0 if mask_bits is None else mask_bits.stride(0),
                              int(planes_only))
        return self.lib.ase_gemm_planes_gemm(self.h, C.byref(p), _stream())

    def run(self, *a, **k):
        self.L.check(self.gemm(*a, **k), 'ase_gemm_planes_gemm')

    def info(self, t):
        """The registry's record of buffer t; scale / inv: what its current planes were written with (backend 2, valid planes)."""
        out = (C.c_int64 * 6)()
        self.scale_buf.fill_(NAN)
        self.L.check(self.lib.ase_gemm_planes_info(self.h, t.data_ptr(), out, self.scale_buf.data_ptr(), _stream()), 'ase_gemm_planes_info')
        s, inv = self.scale_buf.tolist()
        return dict(valid=out[0], stale=out[1], rows=out[2], cols=out[3], ld=out[4], ldp=out[5], scale=s, inv=inv)

    def status(self):
        f = C.c_int()
        self.L.check(self.lib.ase_gemm_planes_status(self.h, C.byref(f), _stream()), 'ase_gemm_planes_status')
        return f.value

    def plane_views(self, t, inf):
        hi, lo = self.planes[t.data_ptr()]
        dt = torch.float16 if self.backend == 2 else torch.float32
        n = inf['rows'] * inf['ldp']
        return [x.view(dt)[:n].view(inf['rows'], inf['ldp'])[:, :inf['cols']] for x in (hi, lo)]

    def consumed(self, t):
        """fp64 of what a consumer of t reads: its fp32 copy, or (hi + lo) / s when the fp32 store was elided (then still all NaN)."""
        inf = self.info(t)
        if not inf['stale']:
            return t.double()
        assert inf['valid'] and bool(torch.isnan(t).all()), ('a planes-only tensor got an fp32 store', inf)
        hi, lo = self.plane_views(t, inf)
        return (hi.double() + lo.double()) / inf['scale']

    def assert_planes_split(self, t, s, what):
        """The planes of the whole buffer t are the exact split of its fp32 contents (at scale s, backend 2)."""
        inf = self.info(t)
        assert inf['valid'] and not inf['stale'], (what, inf)
        assert (inf['rows'], inf['cols'], inf['ld']) == (t.shape[0], t.shape[1], t.stride(0)), (what, inf)
        hi, lo = self.plane_views(t, inf)
        if self.backend == 2:
            assert inf['scale'] == s and inf['inv'] == 1.0 / s, (what, inf, s)
            want = _split_f16(t, s)
        else:
            want = _split_tf32(t)
        _assert_bits_equal(hi, want[0], what + ': hi plane')
        _assert_bits_equal(lo, want[1], what + ': lo plane')


@pytest.fixture
def planes():
    made = []

    def make(backend):
        made.append(Planes(backend))
        return made[-1]
    yield make
    for r in made:
        r.close()


def _randn(g, *shape, scale=1.0):
    return torch.randn(*shape, generator=g, device='cuda') * scale


def _gen(seed):
    return torch.Generator(device='cuda').manual_seed(seed)


# ------------------------------------------------------------------------------------------------ (a) epilogue planes, bit for bit
# (name, M, N, K, tile the plan must pick, options).  Interior tiles of BN = 128 take the fast store phase, everything else (M / N
# tails, BN = 64, N not a multiple of 4) the generic one; 256-row tiles hold two m64 blocks per consumer warpgroup.
EPI_CASES = [
    ('fast_256x128_relu_bits', 4096, 1024, 192, (256, 128), dict(bias=True, act=1, relu_bits=True)),
    ('fast_256x128_fp32_mask_colsum', 4096, 1024, 128, (256, 128), dict(mask='fp32', colsum=True)),
    ('fast_128x128_tanh', 1024, 512, 128, (128, 128), dict(bias=True, act=2, alpha=1.0 / 16)),
    ('fast_128x128_bit_mask', 1024, 512, 96, (128, 128), dict(mask='bits', b_trans=True)),
    ('generic_256_tails_relu', 4040, 1000, 192, (256, 128), dict(bias=True, act=1, relu_bits=True)),
    ('generic_256_tails_bit_mask', 3900, 1000, 96, (256, 128), dict(mask='bits', colsum=True)),
    ('generic_bn64_unaligned_n', 2000, 50, 100, (128, 64), dict(bias=True, act=1, relu_bits=True)),
    ('generic_128_unaligned_n', 700, 1001, 130, (128, 128), dict(bias=True, act=2, alpha=1.0 / 16, b_trans=True)),
    ('fast_128x128_tanh_mask', 1000, 384, 64, (128, 128), dict(mask='tanh')),
]


@pytest.mark.parametrize('tc', TC_BACKENDS)
@pytest.mark.parametrize('case', EPI_CASES, ids=[c[0] for c in EPI_CASES])
def test_epilogue_planes_bit_exact(planes, case, tc):
    from ase_b200 import ops
    name, M, N, K, tile, o = case
    assert ops.gemm_tc_plan(M, N, K, False, 0, tc)[:2] == tile, (name, ops.gemm_tc_plan(M, N, K, False, 0, tc))
    reg = planes(tc)
    Cb = reg.buffer(M, N)
    g = _gen(M + 7 * N + 13 * K)
    b_trans, act, alpha = o.get('b_trans', False), o.get('act', 0), o.get('alpha', 1.0)
    tol = 3e-5 if act == 2 else 1e-5
    prev_max = None
    for call in range(4):
        if call == 3:
            reg.forget()
        reg.begin()
        A = _randn(g, M, K)
        B = _randn(g, K, N) if b_trans else _randn(g, N, K)
        bias = _randn(g, N) if o.get('bias') else None
        mask, mask_src, mask_mode, bits = None, None, 0, None
        if o.get('mask') in ('fp32', 'bits'):
            mask = _randn(g, M, N) > 0
            mask_mode = 1
            mask_src = mask.float() - 0.5 if o['mask'] == 'fp32' else torch.full((M, N), NAN, device='cuda')   # NaN: the bits must be read
            bits = _pack_bits(mask) if o['mask'] == 'bits' else None
        elif o.get('mask') == 'tanh':
            mask_src, mask_mode = _randn(g, M, N).clamp(-0.9, 0.9), 2
        rb = torch.zeros(M, (N + 31) // 32, dtype=torch.int32, device='cuda') if o.get('relu_bits') else None
        cs = torch.zeros(N, device='cuda') if o.get('colsum') else None
        Cb.fill_(NAN)
        reg.run(A, B, Cb, b_trans=b_trans, bias=bias, act=act, mask_src=mask_src, mask_mode=mask_mode, mask_bits=bits, alpha=alpha,
                colsum=cs, relu_bits=rb)
        ref = alpha * _mm(A, B, False, b_trans)
        if bias is not None:
            ref = ref + bias.double()
        ref = torch.relu(ref) if act == 1 else torch.tanh(ref) if act == 2 else ref
        if mask is not None:
            ref = ref * mask.double()
        elif mask_mode == 2:
            ref = ref * (1 - mask_src.double() ** 2)
        _close(Cb, ref, tol, (name, tc, call))
        if rb is not None:
            assert torch.equal(_unpack_bits(rb, N), Cb > 0), (name, call)
        if cs is not None:
            _close(cs, ref.sum(0), 2e-5, (name, tc, call, 'column sums'))
        if tc == 1 or call in (1, 2):
            reg.assert_planes_split(Cb, _site_scale(prev_max) if tc == 2 else None, f'{name} call {call}')
        else:
            assert not reg.info(Cb)['valid'], (name, call)      # the scale is not known yet: the first consumer splits exactly
        prev_max = float(Cb.abs().max())
    assert reg.status() == 0


# ------------------------------------------------------------------------------------------------ (b) the learner's chains
@pytest.mark.parametrize('tc', TC_BACKENDS)
def test_learner_step_chain(planes, tc):
    """One learner step, small and ragged: a 3-layer forward chain (hidden outputs planes-only with ReLU activity bits, consumed
    K-major), the dX chain (weights read MN-major, bit masks, planes-only outputs, fused column sums, a weight sub-view at column 8)
    and the dW GEMMs (split-K accumulation into registered gradient buffers, both operands MN-major from cached planes), then a
    consumer of an accumulated gradient buffer, which must re-split it."""
    from ase_b200 import ops
    reg = planes(tc)
    g = _gen(17)
    Bn, dims = 1100, [100, 200, 136, 24]
    W = [reg.buffer(dims[k + 1], dims[k], _randn(g, dims[k + 1], dims[k], scale=dims[k] ** -0.5)) for k in range(3)]
    bias = [_randn(g, dims[k + 1], scale=0.1) for k in range(3)]
    Y = [reg.buffer(Bn, dims[k + 1]) for k in range(3)]                     # Y[0], Y[1] hidden (planes only), Y[2] the output
    dZ = [reg.buffer(Bn, dims[1]), reg.buffer(Bn, dims[2])]                 # dZ of layers 0 and 1 (planes only)
    dX0 = reg.buffer(Bn, 88)
    G = [reg.buffer(dims[k + 1], dims[k], _randn(g, dims[k + 1], dims[k])) for k in range(3)]
    U = _randn(g, 40, dims[0])
    bits = [torch.zeros(Bn, (dims[k + 1] + 31) // 32, dtype=torch.int32, device='cuda') for k in range(2)]
    split = [ops.gemm_tc_plan(dims[1], dims[0], Bn, True, -1, tc)[2], 3, ops.gemm_tc_plan(dims[3], dims[2], Bn, True, -1, tc)[2]]
    assert split[0] > 1 and split[2] > 1
    prev = {}
    for call in range(4):
        if call == 3:
            reg.forget()
        reg.begin()
        reg.prep_weights(W)
        predicted = tc == 2 and call in (1, 2)
        for t in (Y[0], Y[1], dZ[0], dZ[1], Y[2], dX0):
            t.fill_(NAN)
        X0 = _randn(g, Bn, dims[0])
        dZ3 = _randn(g, Bn, dims[3])
        cs = [torch.zeros(dims[k + 1], device='cuda') for k in range(2)]
        P = torch.zeros(dims[1], 40, device='cuda')
        reg.run(X0, W[0], Y[0], bias=bias[0], act=1, relu_bits=bits[0], planes_only=True)
        reg.run(Y[0], W[1], Y[1], bias=bias[1], act=1, relu_bits=bits[1], planes_only=True)
        reg.run(Y[1], W[2], Y[2], bias=bias[2])
        # backward: the activations are the fp32 masks the learner passes; the bits replace them (and NaN copies must not be read)
        reg.run(dZ3, W[2], dZ[1], b_trans=True, mask_src=Y[1], mask_mode=1, mask_bits=bits[1], planes_only=True, colsum=cs[1])
        reg.run(dZ[1], W[1], dZ[0], b_trans=True, mask_src=Y[0], mask_mode=1, mask_bits=bits[0], planes_only=True, colsum=cs[0])
        reg.run(dZ[0], W[0][:, 8:96], dX0, b_trans=True)
        G0 = [x.double() for x in G]
        reg.run(dZ3, Y[1], G[2], a_trans=True, b_trans=True, accumulate=True, split_k=split[2])
        reg.run(dZ[1], Y[0], G[1], a_trans=True, b_trans=True, accumulate=True, split_k=split[1])
        reg.run(dZ[0], X0, G[0], a_trans=True, b_trans=True, accumulate=True, split_k=split[0])
        for x in G:
            assert not reg.info(x)['valid'], call                     # accumulation leaves the buffer without planes
        reg.run(G[0], U, P)                                             # ... so this consumer splits it again
        torch.cuda.synchronize()
        got = {}
        for name, t in (('Y0', Y[0]), ('Y1', Y[1]), ('dZ0', dZ[0]), ('dZ1', dZ[1])):
            inf = reg.info(t)
            assert inf['stale'] == (1 if predicted else 0), (name, call, inf)
            got[name] = reg.consumed(t)
            if predicted:
                assert inf['scale'] == _site_scale(prev[name]), (name, call, inf, prev[name])
        Wd = [w.double() for w in W]
        ref = torch.relu(X0.double() @ Wd[0].t() + bias[0].double())
        _close(got['Y0'], ref, 1e-5, ('Y0', call))
        assert torch.equal(_unpack_bits(bits[0], dims[1]), got['Y0'] > 0), call
        _close(got['Y1'], torch.relu(got['Y0'] @ Wd[1].t() + bias[1].double()), 1e-5, ('Y1', call))
        assert torch.equal(_unpack_bits(bits[1], dims[2]), got['Y1'] > 0), call
        _close(Y[2], got['Y1'] @ Wd[2].t() + bias[2].double(), 1e-5, ('Y2', call))
        if tc == 1 or predicted:
            reg.assert_planes_split(Y[2], _site_scale(prev.get('Y2')) if tc == 2 else None, f'Y2 call {call}')
        ref = (dZ3.double() @ Wd[2]) * _unpack_bits(bits[1], dims[2]).double()
        _close(got['dZ1'], ref, 1e-5, ('dZ1', call))
        _close(cs[1], ref.sum(0), 2e-5, ('dZ1 column sums', call))
        ref = (got['dZ1'] @ Wd[1]) * _unpack_bits(bits[0], dims[1]).double()
        _close(got['dZ0'], ref, 1e-5, ('dZ0', call))
        _close(cs[0], ref.sum(0), 2e-5, ('dZ0 column sums', call))
        _close(dX0, got['dZ0'] @ Wd[0][:, 8:96], 1e-5, ('dX0', call))
        _close(G[2], G0[2] + dZ3.double().t() @ got['Y1'], 2e-5, ('dW2', call))
        _close(G[1], G0[1] + got['dZ1'].t() @ got['Y0'], 2e-5, ('dW1', call))
        _close(G[0], G0[0] + got['dZ0'].t() @ X0.double(), 2e-5, ('dW0', call))
        _close(P, G[0].double() @ U.double().t(), 1e-5, ('re-split gradient', call))
        prev = {k: float(v.abs().max()) for k, v in got.items()}
        prev['Y2'] = float(Y[2].abs().max())
    assert reg.status() == 0


@pytest.mark.parametrize('tc', TC_BACKENDS)
def test_subview_operands(planes, tc):
    """Consumers of row and column sub-views of one GEMM-written buffer: row offsets (the agent / replay / demo thirds of the
    discriminator input, rows B..2B of the diversity pass) and a column offset of 16 read the cached planes; a column offset of 3
    and a leading dimension other than the declared one fall back to a split of the fp32 copy.  All must match fp64."""
    reg = planes(tc)
    g = _gen(23)
    R, N, K = 300, 136, 72
    H = reg.buffer(3 * R, N)
    W, b = _randn(g, N, K, scale=K ** -0.5), _randn(g, N, scale=0.1)
    V, V16, V3 = _randn(g, 64, N), _randn(g, 64, N - 16), _randn(g, 64, N - 3)
    prev_max = None
    for call in range(4):
        if call == 3:
            reg.forget()
        reg.begin()
        X = _randn(g, 3 * R, K)
        reg.run(X, W, H, bias=b)
        _close(H, X.double() @ W.double().t() + b.double(), 1e-5, ('H', call))
        views = [(H[R:2 * R], V), (H[:R], V), (H[2 * R:], V), (H[R:], V), (H[:, 16:], V16), (H[:, 3:], V3), (H[::2], V)]
        for i, (A, B) in enumerate(views):
            Z = torch.full((A.shape[0], B.shape[0]), NAN, device='cuda')
            reg.run(A, B, Z)
            _close(Z, _mm(A, B), 1e-5, ('view', i, call))
        # the cached planes of H: written by the epilogue at the predicted scale, else split once by the first consumer at the
        # scale of H's own max
        s = _site_scale(prev_max if call in (1, 2) else float(H.abs().max()))
        reg.assert_planes_split(H, s if tc == 2 else None, f'H call {call}')
        prev_max = float(H.abs().max())
    assert reg.status() == 0


def test_prep_weights_split_survive_and_follow(planes):
    """Weights through prep_weights (backend 2): split exactly on the first call; their planes carry their own copy of the scale
    and survive begin_call; after a weight changed, its planes hold the new values (at the scale predicted from the old max), and
    from the following call on the scale follows the new max; forget re-derives it exactly."""
    reg = planes(2)
    g = _gen(29)
    W = [reg.buffer(200, 100, _randn(g, 200, 100)), reg.buffer(72, 200, _randn(g, 72, 200, scale=0.5))]
    X, D = _randn(g, 500, 100), _randn(g, 500, 200)
    split_max = {}
    calls = [('exact', True), ('survive', False), ('changed', True), ('follow', True), ('forget', True)]
    for call, (kind, prep) in enumerate(calls):
        if kind == 'changed':
            old = float(W[0].abs().max())
            W[0].copy_(_randn(g, 200, 100, scale=4.0))          # an optimizer step moved it; its max grew about 4x
            assert _site_scale(W[0].abs().max()) != _site_scale(old)
        if kind == 'forget':
            reg.forget()
        reg.begin()
        if prep:
            reg.prep_weights(W)
        for i, w in enumerate(W):
            s = _site_scale(w.abs().max()) if kind in ('exact', 'forget') else _site_scale(split_max[i])
            reg.assert_planes_split(w, s, f'weight {i} call {call} ({kind})')
        Y = torch.full((500, 200), NAN, device='cuda')
        Z = torch.full((500, 72), NAN, device='cuda')
        Q = torch.full((500, 100), NAN, device='cuda')
        reg.run(X, W[0], Y)                     # K-major
        reg.run(Y, W[1], Z)
        reg.run(D, W[0], Q, b_trans=True)       # MN-major
        _close(Y, X.double() @ W[0].double().t(), 1e-5, ('Y', call))
        _close(Z, Y.double() @ W[1].double().t(), 1e-5, ('Z', call))
        _close(Q, D.double() @ W[0].double(), 1e-5, ('Q', call))
        if prep:
            split_max = {i: float(w.abs().max()) for i, w in enumerate(W)}
    assert reg.status() == 0


@pytest.mark.parametrize('tc', TC_BACKENDS)
def test_planes_of_previous_call_are_resplit(planes, tc):
    """A tensor produced in one call and consumed first thing in the next: its epilogue-written planes refer to a scale slot that
    begin_call has just re-predicted, so they are dropped and the consumer re-splits the fp32 copy.  The tensor grows 4x per call,
    so reading the old planes with the new inverse scale would be 4x off."""
    reg = planes(tc)
    g = _gen(31)
    R, N, K = 300, 136, 96
    Y = reg.buffer(R, N, _randn(g, R, N))                 # written before the first call, as by a non-GEMM kernel
    W, V = _randn(g, N, K, scale=K ** -0.5), _randn(g, 40, N)
    prev_max = None
    for call in range(4):
        if call == 3:
            reg.forget()
        reg.begin()
        if tc == 2 and call > 0:
            assert not reg.info(Y)['valid'], call
        Yc = Y.double()
        Z = torch.full((R, 40), NAN, device='cuda')
        reg.run(Y, V, Z)                                    # first use in this call
        _close(Z, Yc @ V.double().t(), 1e-5, ('consumer of the previous call', call))
        X = _randn(g, R, K, scale=4.0 ** call)
        reg.run(X, W, Y)                                    # produced for the next call
        _close(Y, X.double() @ W.double().t(), 1e-5, ('producer', call))
        if tc == 1 or call in (1, 2):
            reg.assert_planes_split(Y, _site_scale(prev_max) if tc == 2 else None, f'Y call {call}')
        prev_max = float(Y.abs().max())
    assert reg.status() == 0


# ------------------------------------------------------------------------------------------------ errors, never wrong numbers
def test_planes_only_misuse_is_an_error(planes):
    """A planes-only tensor (fp32 store elided) consumed where its planes cannot be used, accumulated into, or read after
    begin_call dropped its planes; and more GEMMs in one call than scale sites.  Each must return an error."""
    from ase_b200 import lib as L
    reg = planes(2)
    g = _gen(37)
    R, N, K = 256, 136, 64
    Y = reg.buffer(R, N)
    X, W, V, V3 = _randn(g, R, K), _randn(g, N, K, scale=K ** -0.5), _randn(g, 32, N), _randn(g, 32, N - 3)
    Z = torch.zeros(R, 32, device='cuda')
    O = torch.zeros(R, N, device='cuda')

    def expect(rc, code, text):
        assert rc == code, (rc, L.lib.ase_last_error())
        assert text in L.lib.ase_last_error().decode(), L.lib.ase_last_error()

    reg.begin()                                                  # call 0 calibrates: the fp32 copy is still stored
    reg.run(X, W, Y, act=1, planes_only=True)
    reg.run(Y, V, Z)
    assert not reg.info(Y)['stale']
    reg.begin()                                                  # call 1: predicted scale, planes only
    Y.fill_(NAN)
    reg.run(X, W, Y, act=1, planes_only=True)
    assert reg.info(Y)['stale']
    expect(reg.gemm(Y[:, 3:], V3, Z), ERR_INVALID, 'elided')                                   # column offset 3: no plane view
    expect(reg.gemm(Y[::2], V, Z[:R // 2]), ERR_INVALID, 'elided')                             # another leading dimension
    expect(reg.gemm(X, W, O, mask_src=Y, mask_mode=1), ERR_INVALID, 'elided')                  # fp32 mask without bits
    expect(reg.gemm(X, W, O, mask_src=Y, mask_mode=2), ERR_INVALID, 'elided')
    expect(reg.gemm(X, W, Y, accumulate=True), ERR_INVALID, 'accumulating into a planes-only tensor')
    Z.fill_(NAN)
    reg.run(Y, V, Z)                                             # the planes themselves are still intact
    _close(Z, reg.consumed(Y) @ V.double().t(), 1e-5, 'after the refused calls')
    _close(reg.consumed(Y), torch.relu(X.double() @ W.double().t()), 1e-5, 'planes-only Y')
    reg.begin()                                                  # call 2: the planes are dropped, and there is no fp32 copy
    expect(reg.gemm(Y, V, Z), ERR_INVALID, 'lost its planes')
    reg.begin(SITES - 6)                                         # two GEMMs fit in the last six sites, a third does not
    reg.run(X, W, O)
    reg.run(X, W, O)
    expect(reg.gemm(X, W, O), ERR_WORKSPACE, 'scale sites')


# ------------------------------------------------------------------------------------------------ the scale window, per site
@pytest.mark.parametrize('factor,flag_now,flag_next', [(64.0, 0, 0), (2.0 ** -13, 0, 0), (512.0, 1, None), (2.0 ** -16, 0, 2)],
                         ids=['x64', 'x2^-13', 'x512', 'x2^-16'])
def test_scale_window(planes, factor, flag_now, flag_next):
    """An input scaled by a power of two between two calls: x64 and 2^-13 fit the predicted scales (no flag, fp64 bar); x512
    overflows (bit 0, in the same call); 2^-16 underflows (bit 1, when the next call starts)."""
    reg = planes(2)
    g = _gen(41)
    R, N, K = 300, 136, 96
    Y = reg.buffer(R, N)
    X0, W, V = _randn(g, R, K), _randn(g, N, K, scale=K ** -0.5), _randn(g, 40, N)
    Z = torch.zeros(R, 40, device='cuda')
    for call, f in enumerate([1.0, 1.0, factor, factor]):
        reg.begin()
        if call == 3:
            assert reg.status() == flag_next, (factor, reg.status())
            break
        X = X0 * f
        reg.run(X, W, Y)
        reg.run(Y, V, Z)
        st = reg.status()
        if call < 2:
            assert st == 0, (call, st)
            continue
        assert st == flag_now, (factor, st)
        if flag_now:
            break
        if factor > 2.0 ** -14:
            _close(Y, X.double() @ W.double().t(), 1e-5, ('Y', factor))
            _close(Z, Y.double() @ V.double().t(), 1e-5, ('Z', factor))


def test_scale_site_that_saw_only_zeros(planes):
    """An output site that only saw zeros keeps scale 0; when data arrives the epilogue must raise bit 1, not write zero planes silently."""
    reg = planes(2)
    g = _gen(43)
    R, N, K = 300, 136, 96
    Y = reg.buffer(R, N)
    W = _randn(g, N, K)
    reg.begin()
    reg.run(torch.zeros(R, K, device='cuda'), W, Y)               # not consumed in this call: the site's scale slot is never set
    assert reg.status() == 0
    reg.begin()
    reg.run(_randn(g, R, K), W, Y)
    assert reg.status() & 2
