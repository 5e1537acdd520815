"""Plain recursive restatement of leaf splitting (volrend_b200/refine.py, DESIGN.md 19) -- TEST INFRASTRUCTURE.

One depth-first walk from the root lists the candidate leaves with their depth; a sort picks the ones to split; a loop
appends one node per split slot.  No vectorisation, so that it shares nothing with the product code but the rules:
  * a candidate is a leaf slot (link 0) of a node reached from the root, at depth < min(max_depth, 23) (root's slots
    are depth 1), with a finite score > 0;
  * the ceil(fraction * n_candidates) candidates with the highest scores are split, ties by the lower slot index;
  * existing nodes keep their index; new nodes are appended in increasing order of the split slot; the split slot's
    link is new_node - its_node; every slot of a new node takes the split slot's row (src), existing slots their own.
"""
import math
import sys

import numpy as np


def refine(child, scores, fraction, max_depth=23):
    """-> (child2 int32 [cap2, 2, 2, 2], src list of the source slot of every output slot)."""
    child = np.asarray(child)
    cap = child.shape[0]
    ch = child.reshape(cap, 8)
    s = np.asarray(scores, np.float32).reshape(cap * 8)
    max_depth = min(int(max_depth), 23)
    cands = []

    def walk(node, depth):
        for o in range(8):
            c = int(ch[node, o])
            if c != 0:
                walk(node + c, depth + 1)
            elif depth < max_depth and math.isfinite(float(s[node * 8 + o])) and float(s[node * 8 + o]) > 0:
                cands.append(node * 8 + o)

    limit = sys.getrecursionlimit()
    sys.setrecursionlimit(max(limit, 1000))
    try:
        walk(0, 1)
    finally:
        sys.setrecursionlimit(limit)
    cands.sort(key=lambda slot: (-float(s[slot]), slot))
    n = math.ceil(fraction * len(cands))
    split = sorted(cands[:n])
    rows = [list(map(int, ch[i])) for i in range(cap)]
    src = list(range(cap * 8))
    for slot in split:
        new = len(rows)
        rows[slot // 8][slot % 8] = new - slot // 8
        rows.append([0] * 8)
        src.extend([slot] * 8)
    return np.array(rows, np.int32).reshape(-1, 2, 2, 2), src
