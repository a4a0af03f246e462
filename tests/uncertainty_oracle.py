"""Segmentation uncertainty over marginal_oracle.Lattice, the definition of the option "uncertainty"
(include/vibrato_b200.h), in float64 with exact (Python int) path costs:

  delta(k -> c)   R(k) + cost(k -> c) - R(c) >= 0, the edge's slack against the prefix minima R (R(EOS) = r_eos);
  entropy         -sum P ln P = ln Z + theta E[cost] = a_eos + theta * sum_edges P(edge) delta(edge),
                  P(k -> c) = exp(a(k) + b(c) - theta delta - a_eos); 0 for an empty sentence or one without a path;
  log_path_prob   -a_eos = ln(exp(-theta min cost) / Z); 0 for an empty sentence, -inf without a path;
  boundary[p]     P(a token of the path ends at character position p) = the sum of the marginals of ends[p], p = 0..n;
                  1 at p = 0 and for the empty sentence's one position, all 0 without a path.

Also the same three values from a brute-force enumeration of every path, and exactly (rationals, with the logarithm
taken in `decimal`) for lattices whose costs are multiples of one unit at theta = ln 2 / unit.  Test infrastructure."""
import decimal
import math
from fractions import Fraction

import numpy as np

import marginal_oracle as mo

NEG = -math.inf


def _forward_backward(lat, theta):
    """(R, a, b, r_eos, a_eos) of marginal_oracle.marginals, for a sentence that has a path."""
    R, a = {(0, 0): 0}, {(0, 0): 0.0}
    for n in lat.nodes[1:]:
        xs = [(R[k] + lat.w(k, n), k) for k in lat.preds(n)]
        R[n] = min(x for x, _ in xs)
        a[n] = mo._lse([a[k] - theta * (x - R[n]) for x, k in xs])
    xs = [(R[k] + lat.w(k, None), k) for k in ((lat.eos_row, i) for i in range(len(lat.ends[lat.eos_row])))]
    r_eos = min(x for x, _ in xs)
    a_eos = mo._lse([a[k] - theta * (x - r_eos) for x, k in xs])
    b = {}
    for n in reversed(lat.nodes):
        terms = [b[c] - theta * (R[n] + lat.w(n, c) - R[c]) for c in lat.succ.get(n[0], []) if n[0] != lat.eos_row]
        if n[0] == lat.eos_row:
            terms.append(-theta * (R[n] + lat.w(n, None) - r_eos))
        b[n] = mo._lse(terms)
    return R, a, b, r_eos, a_eos


def edges(lat):
    """Every edge (k, c) of the lattice, c None for EOS."""
    for k in lat.nodes:
        if k[0] == lat.eos_row:
            yield k, None
        else:
            for c in lat.succ.get(k[0], []):
                yield k, c


def has_path(lat):
    return bool(lat.ends[lat.eos_row])


def uncertainty(lat, theta):
    """(entropy, log_path_prob, boundary list of n + 1 floats) of a non-empty sentence's lattice."""
    n_pos = len(lat.ends)
    if not has_path(lat):
        return 0.0, NEG, [0.0] * n_pos
    R, a, b, r_eos, a_eos = _forward_backward(lat, theta)
    ed = 0.0
    for k, c in edges(lat):
        if c is None:
            delta, bc = R[k] + lat.w(k, None) - r_eos, 0.0
        else:
            delta, bc = R[k] + lat.w(k, c) - R[c], b[c]
        ed += math.exp(a[k] + bc - theta * delta - a_eos) * delta
    prob = {n: math.exp(a[n] + b[n] - a_eos) for n in lat.nodes}
    boundary = [1.0] + [sum(prob[(p, i)] for i in range(len(lat.ends[p]))) for p in range(1, n_pos)]
    return a_eos + theta * ed, -a_eos, boundary


def sentence_uncertainty(bo, sent, theta, bounds=()):
    """(entropy, log_path_prob, boundary) of one sentence (bytes), the empty one included."""
    if not sent:
        return 0.0, 0.0, [1.0]
    return uncertainty(mo.Lattice(bo, sent, bounds), theta)


def batch_uncertainty(bo, sentences, theta, boundaries=None):
    """(entropies float64[n], log_path_probs float64[n], boundary_offsets uint64[n + 1], boundary float64[]), flat like
    BatchResult.entropies / log_path_probs / boundary_offsets / boundary_probs."""
    ent, lpp, bnd = [], [], []
    off = [0]
    for i, s in enumerate(sentences):
        e, l, b = sentence_uncertainty(bo, s, theta, boundaries[i] if boundaries else ())
        ent.append(e)
        lpp.append(l)
        bnd += b
        off.append(len(bnd))
    return (np.array(ent, dtype=np.float64), np.array(lpp, dtype=np.float64), np.array(off, dtype=np.uint64),
            np.array(bnd, dtype=np.float64))


def brute_force(lat, theta):
    """(entropy, log_path_prob, boundary, expected tokens) from the enumeration of every path."""
    paths = mo.all_paths(lat)
    n_pos = len(lat.ends)
    if not paths:
        return 0.0, NEG, [0.0] * n_pos, 0.0
    cmin = min(c for c, _ in paths)
    w = [math.exp(-theta * (c - cmin)) for c, _ in paths]
    z = sum(w)
    ps = [x / z for x in w]
    h = -sum(p * math.log(p) for p in ps if p > 0)
    boundary = [1.0] + [0.0] * (n_pos - 1)
    tokens = 0.0
    for p, (_, nodes) in zip(ps, paths):
        tokens += p * len(nodes)
        for nd in nodes:
            boundary[nd[0]] += p
    return h, math.log(1.0 / z), boundary, tokens


def exact_uncertainty(lat, unit, prec=60):
    """(entropy, log_path_prob) exactly, rounded once to float64, for a lattice whose every edge cost is a multiple
    of `unit`, at theta = ln 2 / unit: an edge of cost k * unit weighs 2^-k, so Z and E[delta] are rationals
    (Fractions over the forward and backward sums), and ln Z is taken in `decimal` at `prec` digits.  With every cost 0
    the weights are path counts, and the values hold at any theta."""
    def k(c):
        q, r = divmod(c, unit)
        assert r == 0, (c, unit)
        return q

    def wt(c):
        return Fraction(1, 2 ** k(c)) if c >= 0 else Fraction(2 ** -k(c))

    f, R = {(0, 0): Fraction(1)}, {(0, 0): 0}
    for n in lat.nodes[1:]:
        f[n] = sum(f[p] * wt(lat.w(p, n)) for p in lat.preds(n))
        R[n] = min(R[p] + lat.w(p, n) for p in lat.preds(n))
    last = [(lat.eos_row, i) for i in range(len(lat.ends[lat.eos_row]))]
    z = sum(f[p] * wt(lat.w(p, None)) for p in last)
    r_eos = min(R[p] + lat.w(p, None) for p in last)
    b = {}
    for n in reversed(lat.nodes):
        if n[0] == lat.eos_row:
            b[n] = wt(lat.w(n, None))
        else:
            b[n] = sum((b[c] * wt(lat.w(n, c)) for c in lat.succ.get(n[0], [])), Fraction(0))
    ed = Fraction(0)  # E[delta] in units
    for kk, c in edges(lat):
        if c is None:
            ed += f[kk] * wt(lat.w(kk, None)) * k(R[kk] + lat.w(kk, None) - r_eos)
        else:
            ed += f[kk] * wt(lat.w(kk, c)) * b[c] * k(R[kk] + lat.w(kk, c) - R[c])
    ed /= z
    with decimal.localcontext() as ctx:
        ctx.prec = prec
        ln2 = decimal.Decimal(2).ln()
        ln_z = decimal.Decimal(z.numerator).ln() - decimal.Decimal(z.denominator).ln()
        a_eos = ln_z + ln2 * k(r_eos)  # ln Z + theta r_eos
        h = a_eos + ln2 * (decimal.Decimal(ed.numerator) / decimal.Decimal(ed.denominator))
        return float(h), float(-a_eos)
