"""Lattice output over BoundedOracle (tests/bounded_oracle.py), the definition of the option "lattice"
(include/vibrato_b200.h):

  nodes  the entries of ends[1..=len] in row order (by end position, then insertion order), BOS left out;
  record (start_word, end, c2b[start_word], c2b[end], word_idx, min_cost), TOKEN_DTYPE like a token;
  link   prev = the sentence-relative index of ends[start_node][min_idx & 0xFFFF], -1 when that is BOS;
         flags = NODE_BEST for the nodes of the best path;
  prob   the node's marginal from tests/marginal_oracle.py (with a theta).

Test infrastructure."""
import numpy as np

from bounded_oracle import TOKEN_DTYPE
import marginal_oracle as mo

LINK_DTYPE = np.dtype([("prev", "<i4"), ("flags", "<u4")])
NODE_BEST = 1


def sentence_lattice(bo, sent, bounds=(), theta=None):
    """(nodes TOKEN_DTYPE, links LINK_DTYPE, probs float list or None) of one sentence (bytes)."""
    if not sent:
        return np.zeros(0, dtype=TOKEN_DTYPE), np.zeros(0, dtype=LINK_DTYPE), ([] if theta else None)
    ends, (eos_row, eos_idx), c2b = bo.lattice(sent, bounds)
    index = {}  # (row, entry) -> node index
    order = []
    for e in range(1, len(ends)):
        for i in range(len(ends[e])):
            index[(e, i)] = len(order)
            order.append((e, i))
    nodes = np.zeros(len(order), dtype=TOKEN_DTYPE)
    links = np.zeros(len(order), dtype=LINK_DTYPE)
    for k, (e, i) in enumerate(order):
        nd = ends[e][i]
        nodes[k] = (nd[1], e, c2b[nd[1]], c2b[e], nd[2], nd[6])
        links[k] = (-1 if nd[0] == 0 else index[(nd[0], nd[5] & 0xFFFF)], 0)
    e, i = eos_row, eos_idx & 0xFFFF  # the best path follows the u16 indices, as BoundedOracle.tokenize does
    while e != 0:
        links[index[(e, i)]]["flags"] = NODE_BEST
        nd = ends[e][i]
        e, i = nd[0], nd[5] & 0xFFFF
    probs = None
    if theta:
        lat = mo.Lattice(bo, sent, bounds)
        prob, _, _ = mo.marginals(lat, theta)
        probs = [prob[n] for n in order]
    return nodes, links, probs


def batch_lattice(bo, sentences, boundaries=None, theta=None):
    """(node_off u64[n+1], nodes, links, probs float64[] or None), flat like BatchResult.node_offsets / nodes /
    node_links / node_probs."""
    parts = [sentence_lattice(bo, s, boundaries[i] if boundaries else (), theta) for i, s in enumerate(sentences)]
    off = np.zeros(len(parts) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(p[0]) for p in parts])
    nodes = np.concatenate([p[0] for p in parts]) if parts else np.zeros(0, dtype=TOKEN_DTYPE)
    links = np.concatenate([p[1] for p in parts]) if parts else np.zeros(0, dtype=LINK_DTYPE)
    probs = np.array([x for p in parts for x in p[2]], dtype=np.float64) if theta else None
    return off, nodes, links, probs
