"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the rollout's counter-based generator: Philox4x32-10 (Salmon, Moraes, Dror, Shaw,
"Parallel random numbers: as easy as 1, 2, 3", SC 2011) with the addressing and the draws documented in include/ase_b200.h, computed in fp64
from the generator's fp32 uniforms.  The checker for the in-kernel draws of ase_policy_sample_rng, ase_latent_update and ase_task_resample.

Addressing: `rng` is the int64 pair {seed, call} read as uint64.  Word block (row, group) of stream `sid` is
    philox4x32_10(counter = (row, group, call mod 2^32, call >> 32), key = (seed mod 2^32, (seed >> 32) ^ (sid * 0x9E3779B1 mod 2^32))).
Draws:
    normals    stream sid,     group = column // 4: Box-Muller on (x, y) and (z, w) -> (a cos, a sin, b cos, b sin), a = sqrt(-2 ln u(x))
    Bernoulli  stream sid + 1, group 0xFFFFFFFF, word x: u_open(x) < p
    randint    stream sid + 1, group 0xFFFFFFFE, word x: lo + x % max(1, hi - lo)
    uniforms   stream sid,     group 0, words x..w through u_open (the task targets)
    latents    normalize(normals) with F.normalize's eps 1e-12
u_closed(x) = (fp32(x >> 8) + 0.5f) * 2^-24 evaluated in fp32: in (0, 1], the Box-Muller input (the top code rounds to 1.0, a valid radius
input).  u_open(x) = min(u_closed(x), 1 - 2^-24): in (0, 1), like torch.rand, for the Bernoulli comparison and the task uniforms."""
import numpy as np

M0, M1 = 0xD2511F53, 0xCD9E8D57           # round multipliers
W0, W1 = 0x9E3779B9, 0xBB67AE85           # key schedule (Weyl) increments
SID_MUL = 0x9E3779B1                      # stream id -> key word 1
GROUP_BERNOULLI, GROUP_RANDINT = 0xFFFFFFFF, 0xFFFFFFFE
MASK32 = np.uint64(0xFFFFFFFF)
ONE_BELOW = np.float32(1.0) - np.float32(2.0 ** -24)          # 0x1.fffffep-1, the largest float32 below 1


def _u32(v):
    return np.asarray(v, dtype=np.uint64) & MASK32


def philox4x32_10(ctr, key):
    """ctr: 4 arrays (or ints) of 32-bit words, key: 2 -> 4 uint64 arrays holding the 32-bit output words (broadcast over the inputs).
    Ten rounds of  (c0, c1, c2, c3) <- (hi(M1 c2) ^ c1 ^ k0, lo(M1 c2), hi(M0 c0) ^ c3 ^ k1, lo(M0 c0)), the key bumped by (W0, W1)
    after each round; the 32x32 -> 64-bit products are exact in uint64."""
    c0, c1, c2, c3 = np.broadcast_arrays(*[_u32(c) for c in ctr])
    k0, k1 = (_u32(k) for k in key)
    m0, m1, w0, w1, s32 = np.uint64(M0), np.uint64(M1), np.uint64(W0), np.uint64(W1), np.uint64(32)
    for _ in range(10):
        p0, p1 = m0 * c0, m1 * c2
        c0, c1, c2, c3 = (p1 >> s32) ^ c1 ^ k0, p1 & MASK32, (p0 >> s32) ^ c3 ^ k1, p0 & MASK32
        k0, k1 = (k0 + w0) & MASK32, (k1 + w1) & MASK32
    return c0, c1, c2, c3


def key_of(seed, sid):
    """(seed, stream id) -> the two key words; seed is an int64 read as uint64 (negative seeds wrap)."""
    s = int(seed) % (1 << 64)
    return s & 0xFFFFFFFF, (s >> 32) ^ ((int(sid) * SID_MUL) % (1 << 32))


def words(seed, call, sid, rows, group):
    """The 4 output words of block (row, group) of draw `call` (int64 read as uint64), stream sid, for every row in `rows`."""
    c = int(call) % (1 << 64)
    return philox4x32_10((np.asarray(rows), group, c & 0xFFFFFFFF, c >> 32), key_of(seed, sid))


def u01_closed(x):
    """fp32 (x >> 8) + 0.5 rounded to fp32, times 2^-24: values in [2^-25, 1]; codes >= 2^23 round half to even, the top code to 1.0."""
    t = (np.asarray(x, dtype=np.uint64) >> np.uint64(8)).astype(np.float32)
    return (t + np.float32(0.5)) * np.float32(2.0 ** -24)


def u01_open(x):
    """u01_closed capped at the largest float32 below 1: values in [2^-25, 1 - 2^-24]."""
    return np.minimum(u01_closed(x), ONE_BELOW)


def normals(seed, call, sid, n, cols):
    """[n, cols] standard normals (fp64 from the fp32 uniforms) of stream sid."""
    rows = np.arange(n)[:, None]
    out = np.empty((n, 4 * ((cols + 3) // 4)))
    for g in range((cols + 3) // 4):
        x, y, z, w = (u01_closed(v).astype(np.float64) for v in words(seed, call, sid, rows[:, 0], g))
        a, b = np.sqrt(-2.0 * np.log(x)), np.sqrt(-2.0 * np.log(z))
        ty, tw = 2.0 * np.pi * y, 2.0 * np.pi * w
        out[:, 4 * g:4 * g + 4] = np.stack([a * np.cos(ty), a * np.sin(ty), b * np.cos(tw), b * np.sin(tw)], axis=-1)
    return out[:, :cols]


def bernoulli(seed, call, sid, p):
    """[n] 0/1 floats: u_open(word x of stream sid + 1, group 0xFFFFFFFF) < p[row] (p compared as float32)."""
    p = np.asarray(p, dtype=np.float32)
    u = u01_open(words(seed, call, int(sid) + 1, np.arange(p.shape[0]), GROUP_BERNOULLI)[0])
    return (u < p).astype(np.float64)


def randint(seed, call, sid, n, lo, hi):
    """[n] int64 in [lo, max(lo + 1, hi)): lo + (word x of stream sid + 1, group 0xFFFFFFFE) % max(1, hi - lo)."""
    x = words(seed, call, int(sid) + 1, np.arange(n), GROUP_RANDINT)[0]
    return int(lo) + (x % np.uint64(max(1, int(hi) - int(lo)))).astype(np.int64)


def uniforms(seed, call, sid, n):
    """[n, 4] float32 uniforms in (0, 1) of stream sid, group 0 (uniform k of an env = its k-th draw)."""
    return np.stack([u01_open(w) for w in words(seed, call, sid, np.arange(n), 0)], axis=-1)


def latents(seed, call, sid, n, dim):
    """[n, dim] normalize(normals) (F.normalize: v / max(||v||, 1e-12))."""
    v = normals(seed, call, sid, n, dim)
    return v / np.maximum(np.linalg.norm(v, axis=-1, keepdims=True), 1e-12)


# ---- the kernels' semantics on top of the draws (fp64) ---------------------------------------------------------------------------------
HALF_LOG_2PI = 0.5 * np.log(2.0 * np.pi)


def policy_sample(mu, logstd, probs, seed, call, sid):
    """ase_policy_sample_rng: a = mu + exp(logstd) * N(0, 1) (stream sid), mask = Bernoulli(probs) (stream sid + 1; all ones when probs is
    None), rows with mask 0 act with mu.  -> (actions, neglogp, sigma, mask, noise), fp64."""
    mu, logstd = np.asarray(mu, np.float64), np.asarray(logstd, np.float64)
    n, a = mu.shape
    z = normals(seed, call, sid, n, a)
    sig = np.exp(logstd)
    mask = np.ones(n) if probs is None else bernoulli(seed, call, sid, probs)
    act = np.where(mask[:, None] == 0.0, mu, mu + sig * z)
    nlp = 0.5 * (z * z).sum(-1) + HALF_LOG_2PI * a + logstd.sum()
    return act, nlp, np.broadcast_to(sig, (n, a)), mask, z


def latent_update(lat, reset_steps, progress, done, smin, smax, seed, call, sid):
    """ase_latent_update: rows with done != 0 get a fresh latent and reset_steps = randint; other rows with reset_steps <= progress get a
    fresh latent and reset_steps += randint; the rest are untouched.  -> (latents fp64, reset_steps int64, touched bool)."""
    lat = np.array(lat, np.float64)
    steps = np.array(reset_steps, np.int64)
    prog, done = np.asarray(progress, np.int64), np.asarray(done) != 0
    n, dim = lat.shape
    upd = ~done & (steps <= prog)
    touched = done | upd
    lat[touched] = latents(seed, call, sid, n, dim)[touched]
    r = randint(seed, call, sid, n, smin, smax)
    steps = np.where(done, r, np.where(upd, steps + r, steps))
    return lat, steps, touched


def task_draws(seed, call, sid, n, params, task):
    """The draws ase_task_resample takes from {seed, call}, stream sid: u [n, 4] float32 and (except for strike) the change-step randint."""
    u = uniforms(seed, call, sid, n)
    steps = None if task == 'strike' else randint(seed, call, sid, n, params['change_steps_min'], params['change_steps_max'])
    return u, steps
