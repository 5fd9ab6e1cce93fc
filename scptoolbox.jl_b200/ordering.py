"""Elimination orderings for the reduced KKT matrix  [dI + G'W^-2G, A'; A, -dI]  of the cone solver.

`stage_order` is the GPU-specific choice: optimal-control subproblems are chains of N stages
coupled only through the dynamics rows (discretization.jl:454-465) and a few global parameters, so
  1. every stage's local variables and local equality rows are eliminated first (N independent
     elimination sub-trees -> wide levels for the level-scheduled LDL'),
  2. the stage-coupling equality rows follow in nested-dissection order over the time axis,
  3. global variables (time dilation, parameter trust region, ...) come last.
Equality rows are always ordered after the variables they touch (their pivot is only -delta
before the first update).  `rcm_order` is the pattern-only fallback.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp


def propagate_labels(var_stage, G):
    """Give unlabelled variables (-2: e.g. L1 epigraph auxiliaries) the stage of their neighbours."""
    lab = np.array(var_stage, dtype=np.int64)
    Gb = (abs(G.tocsr()) > 0).astype(np.int8).tocsr()
    Gc = Gb.tocsc()
    for _ in range(4):
        unk = np.where(lab == -2)[0]
        if unk.size == 0:
            break
        for v in unk:
            rows = Gc.indices[Gc.indptr[v]:Gc.indptr[v + 1]]
            nb = np.unique(np.concatenate([Gb.indices[Gb.indptr[r]:Gb.indptr[r + 1]] for r in rows])) if rows.size else rows
            l = lab[nb] if nb.size else np.array([], dtype=np.int64)
            ls = l[l >= 0]
            if ls.size:
                lab[v] = ls.min()
            elif np.any(l == -1):
                lab[v] = -1
    lab[lab == -2] = -1
    return lab


def _local_min_degree(nodes, adj, A, n):
    """Greedy minimum-degree order of one stage's local nodes (fill tracked inside the stage only).  Equality rows
    become eligible once one of their variables has been eliminated (their pivot is -delta before that)."""
    ladj = {v: set(adj[v]) for v in nodes}
    elim, order, remaining = set(), [], set(nodes)
    rowcols = {v: set(A.indices[A.indptr[v - n]:A.indptr[v - n + 1]].tolist()) for v in nodes if v >= n}
    while remaining:
        best, bd = None, None
        for v in remaining:
            if v >= n and not (rowcols[v] & elim):
                continue
            d = len(ladj[v] - elim)
            if bd is None or d < bd or (d == bd and v < best):
                best, bd = v, d
        if best is None:
            best = min(remaining)
        nb = [w for w in ladj[best] if w not in elim and w in ladj]
        for a_ in nb:
            ladj[a_].update(nb)
            ladj[a_].discard(a_)
        elim.add(best); remaining.discard(best); order.append(best)
    return order


def stage_order(A, G, var_stage, nstages, local_md=True):
    """perm (length n+p): node eliminated k-th; variables 0..n-1, equality rows n..n+p-1.

    var_stage[v]: stage index 0..nstages-1, -1 for global variables, -2 for 'derive from neighbours'.
    local_md: order each stage's local nodes by greedy minimum degree (about halves the fill)."""
    A = A.tocsr(); G = G.tocsr()
    p, n = A.shape
    lab = propagate_labels(var_stage, G)
    rlo = np.full(p, -1, dtype=np.int64)
    rhi = np.full(p, -1, dtype=np.int64)
    for r in range(p):
        l = lab[A.indices[A.indptr[r]:A.indptr[r + 1]]]
        l = l[l >= 0]
        if l.size:
            rlo[r], rhi[r] = l.min(), l.max()
    order = []
    strad = {}
    local_rows = [[] for _ in range(nstages)]
    rest = []
    for r in range(p):
        if rlo[r] < 0:
            rest.append(n + r)
        elif rlo[r] == rhi[r]:
            local_rows[rlo[r]].append(n + r)
        else:
            strad.setdefault((int(rlo[r]), int(rhi[r])), []).append(n + r)
    adj = None
    if local_md:
        Gb = sp.csr_matrix((np.ones(G.nnz, dtype=np.int32), G.indices, G.indptr), shape=G.shape)
        Ab = sp.csr_matrix((np.ones(A.nnz, dtype=np.int32), A.indices, A.indptr), shape=A.shape)
        K = sp.bmat([[Gb.T @ Gb, Ab.T], [Ab, None]], format="csr")
        adj = [set(K.indices[K.indptr[i]:K.indptr[i + 1]].tolist()) - {i} for i in range(n + p)]
    for k in range(nstages):
        nodes = np.where(lab == k)[0].tolist() + local_rows[k]
        order.extend(_local_min_degree(nodes, adj, A, n) if local_md else nodes)
    placed = set()

    def nd(lo, hi):
        if hi <= lo:
            return []
        mid = (lo + hi) // 2
        out = nd(lo, mid) + nd(mid + 1, hi)
        for (a, b), rr in strad.items():
            if a >= lo and b <= hi and a <= mid < b and (a, b) not in placed:
                placed.add((a, b))
                out += rr
        return out

    order.extend(nd(0, nstages - 1))
    order.extend(np.where(lab == -1)[0].tolist())
    order.extend(rest)
    perm = np.array(order, dtype=np.int32)
    assert perm.size == n + p and np.unique(perm).size == n + p
    return perm


def rcm_order(A, G):
    """Pattern-only fallback: reverse Cuthill-McKee on the reduced KKT graph, rows after their variables."""
    from scipy.sparse.csgraph import reverse_cuthill_mckee
    A = A.tocsr()
    p, n = A.shape
    Gb = (abs(G.tocsr()) > 0).astype(np.int8)
    Ab = (abs(A) > 0).astype(np.int8)
    K = sp.bmat([[Gb.T @ Gb + sp.eye(n, dtype=np.int8), Ab.T], [Ab, sp.eye(p, dtype=np.int8)]], format="csr")
    rcm = reverse_cuthill_mckee(K, symmetric_mode=True)
    pos = np.empty(n + p, dtype=np.int64)
    pos[rcm] = np.arange(n + p)
    # push every equality row just after its last variable
    key = pos.astype(np.float64)
    for r in range(p):
        cols = A.indices[A.indptr[r]:A.indptr[r + 1]]
        if cols.size:
            key[n + r] = max(key[n + r], pos[cols].max() + 0.5)
    return np.argsort(key, kind="stable").astype(np.int32)
