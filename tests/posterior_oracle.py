"""Posterior decoding over marginal_oracle.Lattice, the definition of vbt_tokenizer_set_posterior
(include/vibrato_b200.h), in plain float64 operations (Python floats: every multiply, subtract and add rounds to
nearest on its own):

  valid(n)  n has a path to EOS in the integer graph (n ends at EOS's row, or a successor is valid);
  gain(n)   (g1 * p(n)) - 1 with g1 = gamma + 1, p(n) the float32 marginal given for the node;
  sweep     V(0) = 0; for q = 1 .. EOS's row, over the entries e of ends[q] in row order: if e is valid and
            V(s(e)) > -inf, x(e) = V(s(e)) + gain(e); V(q) = max x, A(q) = the first entry that attains it;
  path      A(EOS's row), A(s(that node)), ... back to BOS;
  gain      V(EOS's row): 0 for an empty sentence, -inf without a path.

p is a parameter (a dict node -> float32), so the device's own published marginals can be fed in; node_probs()
derives it from the restatement's own float64 marginals.  Also the left fold of the gains over a path, and a brute
force over every path.  Test infrastructure."""
import math

import numpy as np

import marginal_oracle as mo
from bounded_oracle import TOKEN_DTYPE

NEG = -math.inf


def wrap(x):
    return (x + 2 ** 31) % 2 ** 32 - 2 ** 31


def node_probs(lat, theta):
    """p of every node: the restatement's float64 marginal rounded to float32."""
    prob, _, _ = mo.marginals(lat, theta)
    return {n: np.float32(v) for n, v in prob.items()}


def valid_nodes(lat):
    """The nodes with a path to EOS, from the integer graph."""
    ok = set()
    for n in reversed(lat.nodes):
        if n[0] == lat.eos_row or (n[0] < lat.eos_row and any(c in ok for c in lat.succ.get(n[0], []))):
            ok.add(n)
    return ok


def gain(g1, p):
    return g1 * float(p) - 1.0


def fold(g1, p, path):
    """((0 + gain_1) + gain_2) + ... over the path's nodes (BOS excluded), in order."""
    v = 0.0
    for n in path:
        v = v + gain(g1, p[n])
    return v


def sweep(lat, p, gamma):
    """(path: nodes without BOS in order, V at EOS) of a non-empty sentence's lattice."""
    if not lat.ends[lat.eos_row]:
        return [], NEG
    g1 = gamma + 1.0
    ok = valid_nodes(lat)
    V, A = {0: 0.0}, {}
    for q in range(1, lat.eos_row + 1):
        best, arg = NEG, None
        for i, nd in enumerate(lat.ends[q]):
            n = (q, i)
            vs = V.get(nd[0], NEG)
            if n not in ok or vs == NEG:
                continue
            x = vs + gain(g1, p[n])
            if x > best:
                best, arg = x, n
        V[q], A[q] = best, arg
    path, q = [], lat.eos_row
    while q != 0:
        n = A[q]
        path.append(n)
        q = lat.node(n)[0]
    return path[::-1], V[lat.eos_row]


def records(lat, path):
    """TOKEN_DTYPE records of a path: start_char = start_word, total_cost = the prefix cost (wrapping i32)."""
    out = np.zeros(len(path), dtype=TOKEN_DTYPE)
    prev, cost = (0, 0), 0
    for k, n in enumerate(path):
        nd = lat.node(n)
        cost += lat.w(prev, n)
        out[k] = (nd[1], n[0], lat.c2b[nd[1]], lat.c2b[n[0]], nd[2], wrap(cost))
        prev = n
    return out


def sentence_posterior(bo, sent, gamma, p=None, theta=None, bounds=()):
    """(records, probs float32 list, V at EOS) of one sentence (bytes).  p: dict node -> float32, or None to derive it
    from the restatement's marginals at theta."""
    if not sent:
        return np.zeros(0, dtype=TOKEN_DTYPE), [], 0.0
    lat = mo.Lattice(bo, sent, bounds)
    if not lat.ends[lat.eos_row]:
        return np.zeros(0, dtype=TOKEN_DTYPE), [], NEG
    if p is None:
        p = node_probs(lat, theta)
    path, v = sweep(lat, p, gamma)
    return records(lat, path), [np.float32(p[n]) for n in path], v


def brute_force(lat, p, gamma):
    """(the largest fold over every BOS -> EOS path, the second largest, paths attaining the largest)."""
    g1 = gamma + 1.0
    folds = sorted(((fold(g1, p, path), path) for _, path in mo.all_paths(lat)), key=lambda t: -t[0])
    best = folds[0][0]
    second = next((f for f, _ in folds if f < best), NEG)
    return best, second, [path for f, path in folds if f == best]
