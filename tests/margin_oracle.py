"""Near-best lattices over BoundedOracle (tests/bounded_oracle.py), the definition of the option "lattice_margin"
(include/vibrato_b200.h), in Python ints over marginal_oracle.Lattice:

  F(n)       the least cost of a path from BOS to n, the edge into n included (R of marginal_oracle.marginals);
  G(n)       the least cost of a path from n to EOS, the edges after n; absent without such a path;
  margin(n)  F(n) + G(n) - best, best = the least cost of the sentence;
  kept       every node with G(n) and margin(n) <= D, and every node of the best path (where i32 costs wrap it can
             have a margin > 0); none for an empty sentence or one without a path;
  link       prev = the index in the kept list of the node the full lattice's link names, -1 for BOS, -2 when that
             node was not kept; flags as in the full lattice.

Test infrastructure."""
import numpy as np

import lattice_oracle as lo
import marginal_oracle as mo

MAX_MARGIN = 1 << 62


def forward(lat):
    """F: dict node -> least cost from BOS (BOS included, 0)."""
    F = {(0, 0): 0}
    for n in lat.nodes[1:]:  # ordered by end position: every predecessor ends earlier
        F[n] = min(F[k] + lat.w(k, n) for k in lat.preds(n))
    return F


def backward(lat):
    """G: dict node -> least cost to EOS, for the nodes that have a path there."""
    G = {}
    for n in reversed(lat.nodes):
        if n[0] == lat.eos_row:
            G[n] = lat.w(n, None)
            continue
        xs = [lat.w(n, c) + G[c] for c in lat.succ.get(n[0], []) if c in G]
        if xs:
            G[n] = min(xs)
    return G


def margins(lat):
    """(margin: dict node -> int for the nodes with a path to EOS, best) of a non-empty sentence's lattice; best is
    None (and the dict empty) when the sentence has no path."""
    F, G = forward(lat), backward(lat)
    if (0, 0) not in G:
        return {}, None
    best = G[(0, 0)]
    return {n: F[n] + G[n] - best for n in lat.nodes[1:] if n in G}, best


def kept_nodes(lat, D, best_nodes=()):
    """The kept nodes of a non-empty sentence's lattice as a set of marginal_oracle.Lattice nodes; best_nodes: the
    nodes of the tokenizer's best path."""
    mg, best = margins(lat)
    if best is None:
        return set()
    return {n for n, m in mg.items() if m <= D} | set(best_nodes)


def pruned_lattice(bo, sent, D, bounds=(), theta=None):
    """(nodes TOKEN_DTYPE, links LINK_DTYPE, margins int64, probs float list or None) of one sentence (bytes): the
    kept part of lattice_oracle.sentence_lattice, in its order."""
    nodes, links, probs = lo.sentence_lattice(bo, sent, bounds, theta)
    if not len(nodes):
        return nodes, links, np.zeros(0, dtype=np.int64), probs
    lat = mo.Lattice(bo, sent, bounds)
    mg, _ = margins(lat)
    order = [n for n in lat.nodes if n[0] != 0]  # sentence_lattice's node order
    kept = kept_nodes(lat, D, lat.best_path())
    keep = [k for k, n in enumerate(order) if n in kept]
    new_index = {k: j for j, k in enumerate(keep)}
    out_links = links[keep].copy()
    for j, k in enumerate(keep):
        p = int(links[k]["prev"])
        out_links[j]["prev"] = -1 if p == -1 else new_index.get(p, -2)
    out_margins = np.array([mg[order[k]] for k in keep], dtype=np.int64)
    return nodes[keep].copy(), out_links, out_margins, (None if probs is None else [probs[k] for k in keep])


def batch_pruned_lattice(bo, sentences, D, boundaries=None, theta=None):
    """(node_off u64[n+1], nodes, links, margins int64, probs float64[] or None), flat like BatchResult.node_offsets /
    nodes / node_links / node_margins / node_probs."""
    parts = [pruned_lattice(bo, s, D, boundaries[i] if boundaries else (), theta) for i, s in enumerate(sentences)]
    off = np.zeros(len(parts) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(p[0]) for p in parts])
    nodes = np.concatenate([p[0] for p in parts]) if parts else np.zeros(0, dtype=lo.TOKEN_DTYPE)
    links = np.concatenate([p[1] for p in parts]) if parts else np.zeros(0, dtype=lo.LINK_DTYPE)
    margin = np.concatenate([p[2] for p in parts]) if parts else np.zeros(0, dtype=np.int64)
    probs = np.array([x for p in parts for x in p[3]], dtype=np.float64) if theta else None
    return off, nodes, links, margin, probs
