"""Marginal probabilities over the lattice of BoundedOracle (tests/bounded_oracle.py): forward-backward in float64
with exact (Python int) path costs, the definition of vbt_tokenizer_set_marginals (include/vibrato_b200.h):

  edges  k -> c for every node k of ends[c.start_node], of cost conn(k.right, c.left) + word_cost(c);
         k -> EOS for every node k of the row EOS connects to, of cost conn(k.right, 0);
  P(path) = exp(-theta * cost(path)) / Z,  prob(node) = sum of P over the paths through it,
  path_prob = exp(-theta * min cost) / Z.

Also a brute-force enumeration of every BOS -> EOS path, the large-theta limit (exact counts of minimum-cost
paths), the exact marginals of lattices whose costs are multiples of one unit, and the float32 comparison the device
outputs are held to.  Test infrastructure."""
import math

import numpy as np

NEG = -math.inf


def _lse(xs):
    m = max(xs, default=NEG)
    if m == NEG:
        return NEG
    return m + math.log(sum(math.exp(x - m) for x in xs))


class Lattice:
    """The lattice of one non-empty sentence as nodes (end, index) of BoundedOracle.lattice, with its edges."""

    def __init__(self, bo, sent, bounds=()):
        ends, (self.eos_row, self.best_idx), self.c2b = bo.lattice(sent, bounds)
        self.ends = ends
        self.nodes = [(e, i) for e in range(len(ends)) for i in range(len(ends[e]))]
        self.succ = {}  # start position -> nodes starting there
        for e, row in enumerate(ends):
            for i, nd in enumerate(row):
                if e:
                    self.succ.setdefault(nd[0], []).append((e, i))
        self.bo = bo

    def node(self, n):
        return self.ends[n[0]][n[1]]

    def w(self, k, c):
        """Cost of the edge k -> c (c None: EOS)."""
        right = self.node(k)[4]
        if c is None:
            return self.bo.conn(right, 0)
        nd = self.node(c)
        return self.bo.conn(right, nd[3]) + nd[7]  # the entry's cost, not that of the u16 word_idx

    def preds(self, c):
        s = self.node(c)[0]
        return [(s, i) for i in range(len(self.ends[s]))]

    def best_path(self):
        """The tokenizer's best path (wrapped i32 arithmetic, as the tokens follow it), BOS excluded, in order."""
        out = []
        e, i = self.eos_row, self.best_idx & 0xFFFF  # u16 indices, as BoundedOracle.tokenize follows them
        while e != 0:
            out.append((e, i))
            nd = self.ends[e][i]
            e, i = nd[0], nd[5] & 0xFFFF
        return out[::-1]


def marginals(lat, theta):
    """-> (prob: dict node -> float, path_prob, R(EOS)) by forward-backward relative to the exact prefix minima."""
    R, a = {(0, 0): 0}, {(0, 0): 0.0}
    for n in lat.nodes[1:]:  # ordered by end position: every predecessor ends earlier
        xs = [(R[k] + lat.w(k, n), k) for k in lat.preds(n)]
        R[n] = min(x for x, _ in xs)
        a[n] = _lse([a[k] - theta * (x - R[n]) for x, k in xs])
    last = [(lat.eos_row, i) for i in range(len(lat.ends[lat.eos_row]))]
    xs = [(R[k] + lat.w(k, None), k) for k in last]
    r_eos = min(x for x, _ in xs)
    a_eos = _lse([a[k] - theta * (x - r_eos) for x, k in xs])
    b = {}
    for n in reversed(lat.nodes):
        terms = [b[c] - theta * (R[n] + lat.w(n, c) - R[c]) for c in lat.succ.get(n[0], []) if n[0] != lat.eos_row]
        if n[0] == lat.eos_row:
            terms.append(-theta * (R[n] + lat.w(n, None) - r_eos))
        b[n] = _lse(terms)
    prob = {n: math.exp(a[n] + b[n] - a_eos) for n in lat.nodes}
    return prob, math.exp(-a_eos), r_eos


def all_paths(lat, limit=200000):
    """Every BOS -> EOS path as (exact cost, nodes without BOS)."""
    out = []

    def walk(k, cost, path):
        if len(out) > limit:
            raise RuntimeError("too many paths to enumerate")
        if k[0] == lat.eos_row:
            out.append((cost + lat.w(k, None), path))
        for c in lat.succ.get(k[0], []) if k[0] != lat.eos_row else []:
            walk(c, cost + lat.w(k, c), path + [c])

    walk((0, 0), 0, [])
    return out


def brute_force(lat, theta):
    """(prob, path_prob) from the enumeration of all paths."""
    paths = all_paths(lat)
    cmin = min(c for c, _ in paths)
    weights = [math.exp(-theta * (c - cmin)) for c, _ in paths]
    z = sum(weights)
    prob = {n: 0.0 for n in lat.nodes}
    prob[(0, 0)] = 1.0
    for wgt, (_, p) in zip(weights, paths):
        for n in p:
            prob[n] += wgt / z
    return prob, 1.0 / z


def tie_fractions(lat):
    """The theta -> inf limit: per node, (minimum-cost paths through it) / (all minimum-cost paths), as exact
    fractions from counting DPs."""
    from fractions import Fraction
    R, F = {(0, 0): 0}, {(0, 0): 1}
    for n in lat.nodes[1:]:
        xs = [(R[k] + lat.w(k, n), k) for k in lat.preds(n)]
        R[n] = min(x for x, _ in xs)
        F[n] = sum(F[k] for x, k in xs if x == R[n])
    S, G = {}, {}
    for n in reversed(lat.nodes):
        xs = [(lat.w(n, c) + S[c], c) for c in lat.succ.get(n[0], []) if n[0] != lat.eos_row and c in S]
        if n[0] == lat.eos_row:
            xs.append((lat.w(n, None), None))
        if not xs:
            continue
        S[n] = min(x for x, _ in xs)
        G[n] = sum(1 if c is None else G[c] for x, c in xs if x == S[n])
    total_min = S[(0, 0)]
    n_min = G[(0, 0)]
    return {n: Fraction(F[n] * G[n], n_min) if n in S and R[n] + S[n] == total_min else Fraction(0) for n in lat.nodes}


def exact_marginals(lat, unit, bits=None):
    """(prob: dict node -> float, path_prob) exactly, for a lattice whose every edge cost is a multiple of `unit`, at
    theta = ln 2 / unit: a path of cost k * unit then weighs 2^-k, and every forward and backward sum is a dyadic
    m * 2^e with a Python int m (two sums add at the smaller exponent, so no gcd is taken).  Each value is the exact
    rational f(n) b(n) / Z rounded once to float64 (int / int is correctly rounded, subnormals included).  With every
    cost 0 the weights are path counts, and the result holds at any theta.

    An exact m holds as many bits as the weights of the paths into a node span: about 2 000 per character when costs
    range over i16 at unit 64.  `bits` keeps the leading `bits` bits of every sum instead (truncated; a term more than
    `bits` + 2 bits below the other is dropped), so each value is within (number of sums) * 2^(2 - bits) of the exact
    rational, relative: far below a float64 step for bits = 256."""
    def k(c):
        q, r = divmod(c, unit)
        assert r == 0, (c, unit)
        return q

    def add(acc, m, e):
        if acc is None:
            return m, e
        am, ae = acc
        if bits:
            gap = (e + m.bit_length()) - (ae + am.bit_length())
            if gap < -bits - 2:
                return acc
            if gap > bits + 2:
                return m, e
        m, e = (am + (m << (e - ae)), ae) if e >= ae else ((am << (ae - e)) + m, e)
        if bits and m.bit_length() > bits:
            s = m.bit_length() - bits
            m, e = m >> s, e + s
        return m, e

    def ratio(num, den, e):  # num / den * 2^e, correctly rounded
        return (num << e) / den if e >= 0 else num / (den << -e)

    f, R = {(0, 0): (1, 0)}, {(0, 0): 0}
    for n in lat.nodes[1:]:
        acc = None
        for p in lat.preds(n):
            m, e = f[p]
            acc = add(acc, m, e - k(lat.w(p, n)))
        f[n] = acc
        R[n] = min(R[p] + lat.w(p, n) for p in lat.preds(n))
    z = None
    for i in range(len(lat.ends[lat.eos_row])):
        m, e = f[(lat.eos_row, i)]
        z = add(z, m, e - k(lat.w((lat.eos_row, i), None)))
    r_eos = min(R[(lat.eos_row, i)] + lat.w((lat.eos_row, i), None) for i in range(len(lat.ends[lat.eos_row])))
    b = {}
    for n in reversed(lat.nodes):
        acc = None
        if n[0] == lat.eos_row:
            acc = (1, -k(lat.w(n, None)))
        else:
            for c in lat.succ.get(n[0], []):
                if b[c] is not None:
                    m, e = b[c]
                    acc = add(acc, m, e - k(lat.w(n, c)))
        b[n] = acc
    zm, ze = z
    prob = {n: 0.0 if b[n] is None else ratio(f[n][0] * b[n][0], zm, f[n][1] + b[n][1] - ze) for n in lat.nodes}
    return prob, ratio(1, zm, -k(r_eos) - ze)


F32_ULPS = {"worst": 0}  # the largest float32 ulp distance assert_f32_close has seen in this session


def assert_f32_close(got, exact, ulps=2, what=""):
    """got (float32 array) is within `ulps` float32 steps of every exact value rounded to float32
    (np.float32(float(value))), measured between the bit patterns.  NaN, inf and negative values (-0.0 included) are
    refused on either side; subnormals are compared as they are."""
    got = np.asarray(got)
    assert got.dtype == np.float32, got.dtype
    if not (isinstance(exact, np.ndarray) and exact.dtype == np.float64):
        exact = np.array([float(v) for v in exact], dtype=np.float64)
    exp = exact.astype(np.float32)
    assert got.shape == exp.shape, (what, got.shape, exp.shape)
    if not got.size:
        return
    for name, v in (("got", got), ("expected", exp)):
        bad = ~np.isfinite(v) | np.signbit(v)
        assert not bad.any(), (what, name, int(np.argmax(bad)), v[np.argmax(bad)])
    dist = np.abs(got.view(np.int32).astype(np.int64) - exp.view(np.int32).astype(np.int64))
    i = int(np.argmax(dist))
    F32_ULPS["worst"] = max(F32_ULPS["worst"], int(dist[i]))
    assert dist[i] <= ulps, (what, i, f"{float(got[i])!r} vs {float(exp[i])!r}: {int(dist[i])} ulps")


def sentence_marginals(bo, sent, theta, bounds=()):
    """(token probabilities of the best path, in order; path_prob) of one sentence (bytes)."""
    if not sent:
        return [], 1.0
    lat = Lattice(bo, sent, bounds)
    prob, pp, _ = marginals(lat, theta)
    return [prob[n] for n in lat.best_path()], pp


def batch_marginals(bo, sentences, theta, boundaries=None):
    """(token_probs, path_probs) of a batch, flat like BatchResult.token_probs / path_probs."""
    tp, pp = [], []
    for i, s in enumerate(sentences):
        t, p = sentence_marginals(bo, s, theta, boundaries[i] if boundaries else ())
        tp += t
        pp.append(p)
    return tp, pp
