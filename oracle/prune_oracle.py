"""Plain recursive restatement of weight-based pruning (volrend_b200/prune.py, DESIGN.md 17) -- TEST INFRASTRUCTURE.

One depth-first walk decides every slot, a second one lists the surviving nodes; no vectorisation, so that it shares
nothing with the product code but the rules:
  * a leaf slot is dropped iff not (weight >= thresh), i.e. below thresh or NaN; its data row becomes +0;
  * with collapse, an internal slot whose 8 children are all dropped leaves becomes a dropped leaf (bottom-up); the
    root node always stays;
  * nodes no longer reachable are removed, the others keep their order, child links are relative offsets.
"""
import sys

import numpy as np


def prune(child, data, weights, thresh, collapse=True):
    child = np.asarray(child)
    cap = child.shape[0]
    ch = child.reshape(cap, 8)
    w = np.asarray(weights, np.float32).reshape(cap, 8)
    is_leaf = {}      # (node, octant) -> leaf after pruning
    dropped = {}      # (node, octant) -> dropped leaf

    def decide(node):
        """Decides the slots of `node`; True when all 8 end up dropped leaves."""
        for o in range(8):
            c = int(ch[node, o])
            if c == 0:
                is_leaf[node, o] = True
                dropped[node, o] = not (w[node, o] >= thresh)
            elif decide(node + c) and collapse:
                is_leaf[node, o] = True
                dropped[node, o] = True
            else:
                is_leaf[node, o] = False
                dropped[node, o] = False
        return all(dropped[node, o] for o in range(8))

    limit = sys.getrecursionlimit()
    sys.setrecursionlimit(max(limit, 1000))
    try:
        decide(0)
        kept = []

        def walk(node):
            kept.append(node)
            for o in range(8):
                if not is_leaf[node, o]:
                    walk(node + int(ch[node, o]))

        walk(0)
    finally:
        sys.setrecursionlimit(limit)
    kept.sort()
    new = {n: i for i, n in enumerate(kept)}
    dd = data.shape[-1]
    flat = np.asarray(data).reshape(cap, 8, dd)
    out_child = np.zeros((len(kept), 8), np.int32)
    out_data = np.zeros((len(kept), 8, dd), flat.dtype)
    for n in kept:
        for o in range(8):
            if not is_leaf[n, o]:
                out_child[new[n], o] = new[n + int(ch[n, o])] - new[n]
            if not dropped[n, o]:
                out_data[new[n], o] = flat[n, o]
    return out_child.reshape(-1, 2, 2, 2), out_data.reshape(-1, 2, 2, 2, dd)
