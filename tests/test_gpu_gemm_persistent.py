"""GPU tests of the wgmma GEMM's persistent kernel (gemm_tc_kernel with PERSIST, csrc/gemm_tc.cu): launches whose every tile takes
the fragment store phase run min(tiles, SMs) CTAs that loop over the tiles, with the ring's stage and phase carried from tile to
tile and the column-sum slot alternating by tile.  The tiles and the arithmetic per element are those of the one-tile-per-CTA
kernel, so every output must be bit-identical to it: fp32 C, the hi / lo half planes and the ReLU activity bits of every case
are compared, row by row, with a second run of the same seeded cases in a subprocess whose library is pinned to one tile per
CTA (ASE_TC_DEBUG bit 1024; the library reads the bits once per process).  Column sums (shared + global fp32 atomics, order not
fixed) are held to 1e-6 of an fp64 sum of the stored tensor, and C to the fp64 product at the bars of test_gpu_gemm_planes.py.

Shapes: fewer tiles than the 132 SMs, exactly 132, two waves and two tiles more, and 1024 tiles (7 per SM, 100 left over); both tile
heights; K of a single k-block (64), below one (1, 31) and ragged over several (317); and a ragged M, which is not eligible and
must give the same results through the one-tile-per-CTA kernel.  Options cover all four operand majors, act 0 / 1 / 2, bias,
bit and fp32 masks, the tanh-derivative mask, planes-only outputs through the ase_gemm_planes handle and fp32 C + planes."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAN = float('nan')

# (name, M, N, K, tile the plan must pick)
SHAPES = [
    ('below_sms_128', 1024, 512, 64, (128, 128)),            # 32 tiles, one k-block
    ('equal_sms_128', 4224, 512, 31, (128, 128)),            # 33 x 4 = 132 tiles
    ('above_sms_128', 1792, 2432, 317, (128, 128)),          # 266 tiles = 2 x 132 + 2 (the plan never picks 133 whole tiles)
    ('few_tiles_256', 4096, 1024, 1, (256, 128)),            # 128 tiles of 256 rows
    ('many_tiles_256', 32768, 1024, 128, (256, 128)),        # 1024 tiles = 7 x 132 + 100
    ('ragged_m_256', 4040, 1024, 128, (256, 128)),           # not eligible: the one-tile-per-CTA kernel
]
# planes: C is a registered buffer whose planes the epilogue writes; 'only' also elides the fp32 store.  None: plain ase_gemm
OPTIONS = [
    ('plain', dict(planes=None)),
    ('relu_bias_bits_planes_only', dict(bias=True, act=1, relu_bits=True, planes='only')),
    ('bit_mask_colsum_nt', dict(mask='bits', colsum=True, planes='both', b_trans=True)),
    ('tanh_bias_tn', dict(bias=True, act=2, alpha=1.0 / 16, planes='both', a_trans=True)),
    ('fp32_mask_colsum_tt', dict(mask='fp32', colsum=True, planes='both', a_trans=True, b_trans=True)),
    ('tanh_mask_colsum', dict(mask='tanh', colsum=True, planes=None)),
]
CASES = [(s, o) for s in SHAPES for o in OPTIONS]


def run_cases():
    """Every case once on predicted scales.  Returns {case: {output: row hashes}} and the in-process accuracy failures."""
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from ase_b200 import ops
    import test_gpu_gemm_planes as P
    from test_gpu_gemm_store import _row_hash
    out, bad = {}, []
    for (sname, M, N, K, tile), (oname, o) in CASES:
        name = f'{sname}-{oname}'
        assert ops.gemm_tc_plan(M, N, K, False, 0, 2)[:2] == tile, (name, ops.gemm_tc_plan(M, N, K, False, 0, 2))
        g = P._gen(M + 7 * N + 13 * K + len(oname))
        a_trans, b_trans, act, alpha = o.get('a_trans', False), o.get('b_trans', False), o.get('act', 0), o.get('alpha', 1.0)
        A = P._randn(g, K, M) if a_trans else P._randn(g, M, K)
        B = P._randn(g, K, N) if b_trans else P._randn(g, N, K)
        bias = P._randn(g, N) if o.get('bias') else None
        mask, mask_src, mask_mode, bits = None, None, 0, None
        if o.get('mask') in ('fp32', 'bits'):
            mask = P._randn(g, M, N) > 0
            mask_mode = 1
            mask_src = mask.float() - 0.5 if o['mask'] == 'fp32' else torch.full((M, N), NAN, device='cuda')
            bits = P._pack_bits(mask) if o['mask'] == 'bits' else None
        elif o.get('mask') == 'tanh':
            mask_src, mask_mode = P._randn(g, M, N).clamp(-0.9, 0.9), 2
        rb = torch.zeros(M, (N + 31) // 32, dtype=torch.int32, device='cuda') if o.get('relu_bits') else None
        cs = torch.zeros(N, device='cuda') if o.get('colsum') else None
        ref = alpha * P._mm(A, B, a_trans, b_trans)
        if bias is not None:
            ref = ref + bias.double()
        ref = torch.relu(ref) if act == 1 else torch.tanh(ref) if act == 2 else ref
        if mask is not None:
            ref = ref * mask.double()
        elif mask_mode == 2:
            ref = ref * (1 - mask_src.double() ** 2)
        got = {}
        if o['planes'] is None:                       # plain ase_gemm: fp32 C only
            Cb = torch.full((M, N), NAN, device='cuda')
            ops.gemm(A, B, a_trans, b_trans, bias, act, mask_src, mask_mode, out=Cb, alpha=alpha, backend=2, colsum_out=cs,
                     relu_bits_out=rb, mask_bits=bits)
            value = Cb.double()
            got['C'] = _row_hash(Cb)
        else:
            reg = P.Planes(2)
            Cb = reg.buffer(M, N)
            for call in range(2):                     # call 0 calibrates the scale, call 1 writes the planes with it
                reg.begin()
                Cb.fill_(NAN)
                if cs is not None:
                    cs.zero_()
                reg.run(A, B, Cb, a_trans=a_trans, b_trans=b_trans, bias=bias, act=act, mask_src=mask_src, mask_mode=mask_mode,
                        mask_bits=bits, alpha=alpha, colsum=cs, relu_bits=rb, planes_only=o['planes'] == 'only')
            inf = reg.info(Cb)
            assert inf['valid'] and inf['stale'] == (1 if o['planes'] == 'only' else 0), (name, inf)
            value = reg.consumed(Cb)
            hi, lo = reg.plane_views(Cb, inf)
            got['hi'], got['lo'] = _row_hash(hi), _row_hash(lo)
            if o['planes'] == 'both':
                got['C'] = _row_hash(Cb)
                reg.assert_planes_split(Cb, inf['scale'], name)
            if reg.status() != 0:
                bad.append((name, 'plane status', reg.status()))
            reg.close()
        if rb is not None:
            got['relu_bits'] = _row_hash(rb)
            if not torch.equal(P._unpack_bits(rb, N), value > 0):
                bad.append((name, 'activity bits do not match C > 0'))
        err = float((value - ref).abs().max()) / max(float(ref.abs().max()), 1e-30)
        if not err < (3e-5 if act == 2 else 1e-5):
            bad.append((name, 'C against fp64', err))
        if cs is not None:
            want = value.sum(0)
            err = float((cs.double() - want).abs().max()) / max(float(want.abs().max()), 1e-30)
            if not err < 1e-6:
                bad.append((name, 'column sums against the fp64 sum of C', err))
        out[name] = got
    return out, bad


def test_persistent_kernel_matches_one_tile_per_cta_bit_for_bit(tmp_path):
    assert not int(os.environ.get('ASE_TC_DEBUG', '0')) & (256 | 1024), 'this process must run the persistent kernel'
    mine, bad = run_cases()
    assert not bad, bad
    path = str(tmp_path / 'one_tile_per_cta.pt')
    env = dict(os.environ, ASE_TC_DEBUG=str(int(os.environ.get('ASE_TC_DEBUG', '0')) | 1024),
               PYTHONPATH=os.pathsep.join([ROOT] + [p for p in os.environ.get('PYTHONPATH', '').split(os.pathsep) if p]))
    r = subprocess.run([sys.executable, '-s', os.path.abspath(__file__), path], env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    other = torch.load(path)
    assert sorted(other) == sorted(mine)
    diff = []
    for name, outs in mine.items():
        assert sorted(outs) == sorted(other[name]), name
        for k, h in outs.items():
            rows = (h != other[name][k]).nonzero().flatten()
            if rows.numel():
                diff.append((name, k, f'{rows.numel()} rows differ, first {int(rows[0])}'))
    assert not diff, diff


if __name__ == '__main__':      # the one-tile-per-CTA run of the test above
    res, failures = run_cases()
    assert not failures, failures
    torch.save(res, sys.argv[1])
