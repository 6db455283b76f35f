"""Micro-benchmark of ase_gemm over the learner's shapes (CUDA events, warm, L2 flushed between reps by a 256 MB write).
  python tools/bench_gemm.py [backend]                 K / M sweeps and the dX / dW shapes
  python tools/bench_gemm.py [backend] --minibatch     the 54 GEMMs of one config-3 minibatch (ASE pre-train, B = 16384,
                                                       Ba = 4096): per shape the tile plan, kernel time, algorithmic TFLOP/s,
                                                       operand bytes the CTAs load and their rate, and the same shape with
                                                       the tile height pinned to 128 rows (ASE_TC_DEBUG bit 512, in a
                                                       subprocess: the library reads the bits once per process)
  python tools/bench_gemm.py [backend] --minibatch --store-share
                                                       the second column is the same shape with the store phase dropped
                                                       (ASE_TC_DEBUG bit 1) instead: what the store phase costs per shape
  python tools/bench_gemm.py [backend] --minibatch --persistent
                                                       the second column is the same shape on the one-tile-per-CTA kernel
                                                       (ASE_TC_DEBUG bit 1024) instead of the persistent one"""
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from ase_b200 import ops, lib as L

args = [a for a in sys.argv[1:] if not a.startswith('--')]
backend = int(args[0]) if args else 1
flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device='cuda')


def plan(M, N, K, accumulate, split_k):
    """(tile rows, tile cols, splits) the library will launch, or None for a library without the plan query."""
    if not hasattr(L.lib, 'ase_gemm_tc_plan'):
        return None
    bm, bn, s = C.c_int(), C.c_int(), C.c_int()
    L.check(L.lib.ase_gemm_tc_plan(M, N, K, int(accumulate), split_k, backend, C.byref(bm), C.byref(bn), C.byref(s)), 'ase_gemm_tc_plan')
    return bm.value, bn.value, s.value


def operand_bytes(M, N, K, bm, bn):
    """hi + lo plane bytes of A and B that the CTAs of one launch load: every tile reads its rows and columns over all of K
    (split-K divides K between CTAs, not the sum); 128-byte k-blocks."""
    kb = -(-K // (64 if backend == 2 else 32))
    tiles = -(-M // bm) * -(-N // bn)
    return tiles * kb * 2 * (bm + bn) * 128


def measure(M, N, K, a_trans, b_trans, accumulate=False, split_k=0, reps=5, bias=False):
    A = torch.randn((K, M) if a_trans else (M, K), device='cuda')
    B = torch.randn((K, N) if b_trans else (N, K), device='cuda')
    out = torch.zeros(M, N, device='cuda')
    bias_t = torch.randn(N, device='cuda') if bias else None
    ts, kts = [], []
    for r in range(reps + 2):
        flush.zero_()
        L.lib.ase_gemm_tc_profile(1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        ops.gemm(A, B, a_trans, b_trans, bias_t, 1 if bias else 0, out=out, accumulate=accumulate, split_k=split_k, backend=backend)
        e1.record()
        torch.cuda.synchronize()
        ms, n, fl = C.c_double(), C.c_int64(), C.c_double()
        L.lib.ase_gemm_tc_profile_read(C.byref(ms), C.byref(n), C.byref(fl))
        if r >= 2:
            ts.append(e0.elapsed_time(e1)); kts.append(ms.value)
    L.lib.ase_gemm_tc_profile(0)
    return sorted(ts)[len(ts) // 2], sorted(kts)[len(kts) // 2]


def timeit(M, N, K, a_trans, b_trans, accumulate=False, split_k=0, reps=5, **kw):
    t, kt = measure(M, N, K, a_trans, b_trans, accumulate, split_k, reps, kw.get('bias', False))
    fl = 2.0 * M * N * K
    print(f"M={M:6d} N={N:5d} K={K:6d} at={int(a_trans)} bt={int(b_trans)} acc={int(accumulate)} sk={split_k:2d}  total {t*1e3:8.1f} us  "
          f"main kernel {kt*1e3:8.1f} us  {fl/kt/1e9 if kt else 0:7.1f} TFLOP/s (kernel)  {fl/t/1e9:7.1f} TFLOP/s (with prep)")


# One config-3 minibatch (ase_learner_calc_gradients, learner.cu), Ra = 2B rows for the actor (diversity bonus), 3 Ba for the
# discriminator.  (name, M, N, K, a_trans, b_trans, accumulate, split_k, bias): forward layers Y = X W^T (+ bias), dX = dZ W,
# dW += dZ^T X with the learner's split-K (-1: the plan's choice), the gradient-penalty chain.
def minibatch_shapes(B=16384, Ba=4096):
    Ra, R3, Z, IN0, AMP = 2 * B, 3 * Ba, 64, 317, 1400
    s = []
    fwd = lambda n, M, N, K: s.append((n, M, N, K, False, False, False, 0, True))
    dx = lambda n, M, N, K: s.append((n, M, N, K, False, True, False, 0, False))
    dw = lambda n, M, N, K: s.append((n, M, N, K, True, True, True, -1, False))
    nt = lambda n, M, N, K: s.append((n, M, N, K, False, False, False, 0, False))
    fwd('style0', Ra, 512, Z); fwd('style1', Ra, 256, 512); fwd('style_dense', Ra, Z, 256)
    fwd('actor0', Ra, 1024, IN0); fwd('actor1', Ra, 1024, 1024); fwd('actor2', Ra, 512, 1024); fwd('mu', Ra, 31, 512)
    fwd('critic0', B, 1024, IN0); fwd('critic1', B, 1024, 1024); fwd('critic2', B, 512, 1024); fwd('value', B, 1, 512)
    fwd('disc0', R3, 1024, AMP); fwd('disc1', R3, 1024, 1024); fwd('disc2', R3, 512, 1024); fwd('logit', R3, 1, 512)
    fwd('enc', Ba, Z, 512)
    dw('dW mu', 31, 512, Ra); dx('dX mu', Ra, 512, 31)
    dw('dW actor2', 512, 1024, Ra); dx('dX actor2', Ra, 1024, 512); dw('dW actor1', 1024, 1024, Ra); dx('dX actor1', Ra, 1024, 1024)
    dw('dW actor0', 1024, IN0, Ra)
    dx('dX style cols', Ra, Z, 1024); dw('dW style_dense', Z, 256, Ra); dx('dX style_dense', Ra, 256, Z)
    dw('dW style1', 256, 512, Ra); dx('dX style1', Ra, 512, 256); dw('dW style0', 512, Z, Ra)
    dw('dW value', 1, 512, B); dx('dX value', B, 512, 1)
    dw('dW critic2', 512, 1024, B); dx('dX critic2', B, 1024, 512); dw('dW critic1', 1024, 1024, B); dx('dX critic1', B, 1024, 1024)
    dw('dW critic0', 1024, IN0, B)
    dw('dW logit', 1, 512, R3); dw('dW enc', Z, 512, Ba); dx('dX logit', R3, 512, 1)
    s.append(('dX enc (acc)', Ba, 512, Z, False, True, True, 1, False))
    dw('dW disc2', 512, 1024, R3); dx('dX disc2', R3, 1024, 512); dw('dW disc1', 1024, 1024, R3); dx('dX disc1', R3, 1024, 1024)
    dw('dW disc0', 1024, AMP, R3)
    dx('gp U1', Ba, 1024, 512); dx('gp U0', Ba, 1024, 1024); dx('gp G', Ba, AMP, 1024); dw('gp dW0', 1024, AMP, Ba)
    nt('gp Ubar0', Ba, 1024, AMP); dw('gp dW1', 1024, 1024, Ba); nt('gp Ubar1', Ba, 1024, 1024)
    dw('gp dW2', 512, 1024, Ba); nt('gp Ubar2', Ba, 512, 1024)
    assert len(s) == 54
    return s


def minibatch_rows():
    rows = []
    for (name, M, N, K, at, bt, acc, sk, bias) in minibatch_shapes():
        p = plan(M, N, K, acc, sk)
        if sk < 0:      # the learner passes the plan's split count explicitly; a library without the plan uses the old SIMT-style rule
            sk = p[2] if p else 1
        _, kt = measure(M, N, K, at, bt, acc, sk, bias=bias)
        bm, bn = (p[0], p[1]) if p else (128, 128 if N > 64 else 64)
        splits = p[2] if p else (sk if acc and sk > 1 else 1)
        rows.append(dict(name=name, M=M, N=N, K=K, plan=p, split_k=sk, us=kt * 1e3, tflops=2.0 * M * N * K / kt / 1e9,
                         bytes=operand_bytes(M, N, K, bm, bn), ctas=-(-M // bm) * -(-N // bn) * splits))
    return rows


if '--minibatch' in sys.argv:
    rows = minibatch_rows()
    if '--json' in sys.argv:
        print(json.dumps(rows))
        sys.exit(0)
    other_bit, other = ((1, 'no store') if '--store-share' in sys.argv else (1024, 'tile/CTA') if '--persistent' in sys.argv
                        else (512, 'pinned 128'))
    env = dict(os.environ, ASE_TC_DEBUG=str(int(os.environ.get('ASE_TC_DEBUG', '0')) | other_bit))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), str(backend), '--minibatch', '--json'], env=env, capture_output=True, text=True)
    pinned = json.loads(r.stdout.strip().splitlines()[-1]) if r.returncode == 0 else None
    if pinned is None:
        sys.stderr.write(r.stderr)
    print(f"# backend {backend}, {torch.cuda.get_device_name()}; operand bytes = hi/lo plane bytes all CTAs load per launch")
    print(f"{'gemm':16s} {'M':>6s} {'N':>5s} {'K':>6s}  {'plan':>11s} {'us':>8s} {'TFLOP/s':>8s} {'GB':>6s} {'TB/s':>5s}  |"
          f" {other:>11s} {'us':>8s} {'TFLOP/s':>8s} {'GB':>6s} {'TB/s':>5s}")
    tot = [0.0, 0.0, 0.0, 0.0]
    for i, a in enumerate(rows):
        fmt = lambda x: (f"{x['plan'][0]}x{x['plan'][1]}/{x['plan'][2]}" if x['plan'] else '-') + \
            f" {x['us']:8.1f} {x['tflops']:8.1f} {x['bytes']/1e9:6.3f} {x['bytes']/x['us']/1e6:5.2f}"
        line = f"{a['name']:16s} {a['M']:6d} {a['N']:5d} {a['K']:6d}  {fmt(a)}"
        tot[0] += a['us']; tot[1] += a['bytes']
        if pinned:
            b = pinned[i]
            line += f"  | {fmt(b)}"
            tot[2] += b['us']; tot[3] += b['bytes']
        print(line)
    fl = sum(2.0 * a['M'] * a['N'] * a['K'] for a in rows)
    print(f"# minibatch: {tot[0]/1e3:.3f} ms, {fl/tot[0]/1e6:.1f} TFLOP/s, {tot[1]/1e9:.2f} GB operands, {sum(a['ctas'] for a in rows)} CTAs"
          + (f"  | {other}: {tot[2]/1e3:.3f} ms, {fl/tot[2]/1e6:.1f} TFLOP/s, {tot[3]/1e9:.2f} GB operands, "
             f"{sum(b['ctas'] for b in pinned)} CTAs" if pinned else ''))
    sys.exit(0)

print("# forward-like (NT), K sweep at M=32768 N=1024")
for K in (64, 128, 256, 320, 512, 1024, 2048):
    timeit(32768, 1024, K, False, False, bias=True)
print("# M sweep at N=1024 K=1024")
for M in (4096, 8192, 16384, 32768):
    timeit(M, 1024, 1024, False, False, bias=True)
print("# dX-like (B transposed)")
timeit(32768, 1024, 1024, False, True)
timeit(12288, 1400, 1024, False, True)
print("# dW-like (both transposed, split-K accumulate)")
for sk in (1, 2, 5, 10):
    timeit(1024, 1024, 32768, True, True, accumulate=True, split_k=sk)
timeit(1024, 1400, 12288, True, True, accumulate=True, split_k=4)
timeit(512, 1024, 32768, True, True, accumulate=True, split_k=10)
