"""Segmentation sampling over the lattice of BoundedOracle (tests/bounded_oracle.py, tests/marginal_oracle.py), the
definition of vbt_tokenizer_set_sampling (include/vibrato_b200.h):

  Philox4x32-10 with the standard constants; key (seed & 0xFFFFFFFF, seed >> 32), counter (t, j, i, 0) for draw step
  t (0 at EOS) of sample j of sentence i; u = ((x0 >> 5) * 2^26 + (x1 >> 6)) * 2^-53.
  A walk starts at EOS and repeats until BOS.  At node c (EOS: left id 0, word cost 0), over the entries k of the row c
  starts at, in row order: x_k = R(k) + conn(right(k), left(c)) + wcost(c), r = min x_k, t_k = a(k) - theta (x_k - r),
  m = max t_k, w_k = exp(t_k - m); the first k whose running float64 sum exceeds u * S (S the whole sum), else the
  last k with w_k > 0.
  Records as the tokens', total_cost the path's prefix cost through the token wrapped to i32.

A draw is *ambiguous* when some running sum lies within 1e-9 * S of u * S: the device's exp and log-sum-exp may
round differently from Python's there, so a sample is compared only up to its first ambiguous draw.
Test infrastructure."""
import math

import numpy as np

from bounded_oracle import TOKEN_DTYPE
import marginal_oracle as mo

M32 = 0xFFFFFFFF
AMBIGUOUS = 1e-9


def philox4x32_10(ctr, key):
    """Philox4x32-10 of counter (4 words) under key (2 words) -> 4 words."""
    c0, c1, c2, c3 = ctr
    k0, k1 = key
    for r in range(10):
        if r:
            k0 = (k0 + 0x9E3779B9) & M32
            k1 = (k1 + 0xBB67AE85) & M32
        p0 = 0xD2511F53 * c0
        p1 = 0xCD9E8D57 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0) & M32, p1 & M32, ((p0 >> 32) ^ c3 ^ k1) & M32, p0 & M32
    return c0, c1, c2, c3


def uniform(seed, t, j, i):
    """The u of draw step t of sample j of sentence i."""
    x = philox4x32_10((t & M32, j & M32, i & M32, 0), (seed & M32, (seed >> 32) & M32))
    return ((x[0] >> 5) * 67108864.0 + (x[1] >> 6)) * (1.0 / 9007199254740992.0)


def wrap32(v):
    v &= M32
    return v - (1 << 32) if v & 0x80000000 else v


def forward(lat, theta):
    """(R, a, r_eos): exact least costs and forward log weights relative to them, as marginal_oracle.marginals."""
    R, a = {(0, 0): 0}, {(0, 0): 0.0}
    for n in lat.nodes[1:]:
        xs = [(R[k] + lat.w(k, n), k) for k in lat.preds(n)]
        R[n] = min(x for x, _ in xs)
        a[n] = mo._lse([a[k] - theta * (x - R[n]) for x, k in xs])
    r_eos = min(R[(lat.eos_row, i)] + lat.w((lat.eos_row, i), None) for i in range(len(lat.ends[lat.eos_row])))
    return R, a, r_eos


def walk(lat, fw, theta, seed, i, j):
    """One sampled path: (nodes BOS excluded in order, index of the first ambiguous draw or None)."""
    R, a, r_eos = fw
    row, left, wc, r = lat.eos_row, 0, 0, r_eos
    out, amb, t = [], None, 0
    while row != 0:
        ks = [(row, k) for k in range(len(lat.ends[row]))]
        xs = [R[k] + lat.bo.conn(lat.node(k)[4], left) + wc for k in ks]
        ts = [a[k] - theta * (x - r) for k, x in zip(ks, xs)]
        m = max(ts)
        ws = [math.exp(tk - m) for tk in ts]
        S = 0.0
        for w in ws:
            S += w
        target = uniform(seed, t, j, i) * S
        cum, pick, last_pos = 0.0, None, None
        for k, w in enumerate(ws):
            cum += w
            if abs(cum - target) <= AMBIGUOUS * S and amb is None:
                amb = t
            if w > 0:
                last_pos = k
            if cum > target and pick is None:
                pick = k
        if pick is None:
            pick = last_pos
        c = ks[pick]
        out.append(c)
        nd = lat.node(c)
        row, left, wc, r = nd[0], nd[3], nd[7], R[c]
        t += 1
    return out[::-1], amb


def path_cost(lat, path):
    """Exact cost of a path (nodes BOS excluded, in order), the EOS edge included."""
    prev, cost = (0, 0), 0
    for n in path:
        cost += lat.w(prev, n)
        prev = n
    return cost + lat.w(prev, None) if path else 0


def records(lat, path):
    """TOKEN_DTYPE records of a sampled path: as the tokens', total_cost the wrapped prefix cost."""
    out, prev, prefix = [], (0, 0), 0
    for n in path:
        prefix += lat.w(prev, n)
        nd = lat.node(n)
        out.append((nd[1], n[0], lat.c2b[nd[1]], lat.c2b[n[0]], nd[2], wrap32(prefix)))
        prev = n
    return np.array(out, dtype=TOKEN_DTYPE)


def sentence_samples(bo, sent, n, theta, seed, i, bounds=()):
    """The n samples of sentence i (bytes) as [(records, path, first ambiguous draw or None)]."""
    if not sent:
        return [(np.zeros(0, dtype=TOKEN_DTYPE), [], None) for _ in range(n)]
    lat = mo.Lattice(bo, sent, bounds)
    if not lat.ends[lat.eos_row]:
        return [(np.zeros(0, dtype=TOKEN_DTYPE), [], None) for _ in range(n)]
    fw = forward(lat, theta)
    out = []
    for j in range(n):
        path, amb = walk(lat, fw, theta, seed, i, j)
        out.append((records(lat, path), path, amb))
    return out
