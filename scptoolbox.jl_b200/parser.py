"""Host-side conic 'parser' of the GPU path: the mirror of src/parser/{program,constraint,cone,cost}.jl.

The reference rebuilds a JuMP model every SCP iteration (ptr.jl:470-478).  Here the subproblem is
built ONCE, symbolically: a coefficient is not a number but a `Lin` -- a linear combination of
*sources*, i.e. per-seed quantities that live on the device and change every iteration (the DLTV
blocks A_k, B_k, ..., the linearised constraint Jacobians, the reference trajectory).  Compiling the
template yields
  * the batch-shared sparsity pattern of (A, G) and the cone partition for scpb_cone_setup, and
  * one sparse matrix W with   [Avals; Gvals; c; b; h] = W @ src   for every seed,
so that "formulating" an iteration on the GPU is a single pattern-shared SpMV (kernel K6).

Cone semantics follow src/parser/cone.jl:36-47; L1 / LINF are lowered like MathOptInterface's
NormOneBridge / NormInfinityBridge (the path JuMP takes for ECOS).
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp


class Lin:
    """sum_t w_t * src[t]; source 0 is the constant 1."""
    __slots__ = ("t",)

    def __init__(self, t=None):
        self.t = t if t is not None else {}

    @staticmethod
    def const(v):
        v = float(v)
        return Lin({0: v} if v != 0.0 else {})

    @staticmethod
    def src(idx, w=1.0):
        return Lin({int(idx): float(w)})

    @staticmethod
    def lift(v):
        return v if isinstance(v, Lin) else Lin.const(v)

    def is_zero(self):
        return not self.t

    def __add__(self, o):
        o = Lin.lift(o)
        t = dict(self.t)
        for k, v in o.t.items():
            nv = t.get(k, 0.0) + v
            if nv == 0.0:
                t.pop(k, None)
            else:
                t[k] = nv
        return Lin(t)

    __radd__ = __add__

    def __neg__(self):
        return Lin({k: -v for k, v in self.t.items()})

    def __sub__(self, o):
        return self + (-Lin.lift(o))

    def __rsub__(self, o):
        return Lin.lift(o) - self

    def __mul__(self, a):
        a = float(a)
        return Lin({k: v * a for k, v in self.t.items()}) if a != 0.0 else Lin()

    __rmul__ = __mul__


class Expr:
    """const + sum_v coef_v * z_v with Lin coefficients."""
    __slots__ = ("t", "c")

    def __init__(self, t=None, c=None):
        self.t = t if t is not None else {}
        self.c = c if c is not None else Lin()

    @staticmethod
    def lift(v):
        if isinstance(v, Expr):
            return v
        return Expr(None, Lin.lift(v))

    def __add__(self, o):
        o = Expr.lift(o)
        t = dict(self.t)
        for k, v in o.t.items():
            t[k] = t[k] + v if k in t else v
        return Expr(t, self.c + o.c)

    __radd__ = __add__

    def __neg__(self):
        return Expr({k: -v for k, v in self.t.items()}, -self.c)

    def __sub__(self, o):
        return self + (-Expr.lift(o))

    def __rsub__(self, o):
        return Expr.lift(o) - self

    def __mul__(self, a):
        if isinstance(a, Lin):
            return self.scale_lin(a)
        a = float(a)
        if a == 0.0:
            return Expr()
        return Expr({k: v * a for k, v in self.t.items()}, self.c * a)

    __rmul__ = __mul__

    def __truediv__(self, a):
        return self * (1.0 / float(a))

    def is_const_coef(self):
        return all(set(v.t) <= {0} for v in self.t.values()) and set(self.c.t) <= {0}

    def scale_lin(self, L: Lin):
        """Lin * Expr; the expression must have constant coefficients (bilinear terms do not occur:
        device-computed blocks always multiply affinely *scaled variables*, block.jl:368-397)."""
        assert self.is_const_coef(), "product of two source-dependent quantities"
        out = {}
        for k, v in self.t.items():
            out[k] = L * v.t.get(0, 0.0)
        return Expr(out, L * self.c.t.get(0, 0.0))


def matvec(M, v):
    """M: 2-D array of Lin / float (None or 0 = structural zero); v: vector of Expr."""
    out = []
    for i in range(len(M)):
        e = Expr()
        row = M[i]
        for j in range(len(row)):
            m = row[j]
            if m is None or (not isinstance(m, Lin) and m == 0.0):
                continue
            e = e + (v[j] * m if not isinstance(m, Lin) else v[j].scale_lin(m))
        out.append(e)
    return out


class ConicTemplate:
    """Symbolic ConicProgram (program.jl:63-76): variables, cone rows, cost -- with Lin coefficients."""

    def __init__(self, nsrc: int, l1_block: int = 0):
        self.nsrc = nsrc
        # l1_block > 0: lower |x|_1 <= t through partial sums of l1_block epigraph variables (an equivalent
        # program whose normal-equation matrix has no dense (dim x dim) block; 0 = MOI's NormOneBridge form)
        self.l1_block = int(l1_block)
        self.nvar = 0
        self.blocks = {}
        self.var_stage = []       # stage label per variable (-1 global, -2 derive from neighbours)
        self.eq, self.ineq, self.socs = [], [], []
        self.cost = Expr()
        self.sq_log = {}          # epigraph variable of a sumsq -> its squared rows (GuSTO evaluates them on the device)

    def new_variable(self, shape, name, S=None, c=None, stage=None):
        """@new_variable + @scale: returns Expr array in physical units x = S*xh + c.
        stage: 'col' (column index is the stage), 'idx' (vector index is the stage), int, or None (global)."""
        shape = (shape,) if isinstance(shape, int) else tuple(shape)
        n = int(np.prod(shape))
        off = self.nvar
        self.nvar += n
        self.blocks[name] = (off, shape)
        arr = np.empty(shape, dtype=object)
        for i in range(n):
            idx = np.unravel_index(i, shape, order="F")
            e = Expr({off + i: Lin.const(1.0)})
            if S is not None:
                e = e * float(S[idx[0]]) + float(c[idx[0]])
            arr[idx] = e
            if stage == "col":
                self.var_stage.append(int(idx[1]))
            elif stage == "idx":
                self.var_stage.append(int(idx[0]))
            elif stage is None:
                self.var_stage.append(-1)
            elif hasattr(stage, "__len__"):
                self.var_stage.append(int(stage[i]))
            else:
                self.var_stage.append(int(stage))
        return arr

    def _aux(self, n, stage):
        off = self.nvar
        self.nvar += n
        self.var_stage.extend([stage] * n)
        return [Expr({off + i: Lin.const(1.0)}) for i in range(n)]

    # cones (cone.jl:36-47) -------------------------------------------------
    def zero(self, exprs, name=""):
        self.eq.extend(Expr.lift(e) for e in exprs)

    def nonpos(self, exprs, name=""):
        self.ineq.extend(Expr.lift(e) for e in exprs)

    def l1(self, exprs, name="", stage=-2):
        t, xs = Expr.lift(exprs[0]), [Expr.lift(e) for e in exprs[1:]]
        y = self._aux(len(xs), stage)
        for xi, yi in zip(xs, y):
            self.ineq.append(xi - yi)
            self.ineq.append(-xi - yi)
        blk = self.l1_block
        if blk > 0 and len(y) > blk + 1:
            parts = []
            for j in range(0, len(y), blk):
                b = self._aux(1, stage)[0]
                tot = Expr()
                for yi in y[j:j + blk]:
                    tot = tot + yi
                self.ineq.append(tot - b)
                parts.append(b)
            y = parts
        tot = Expr()
        for yi in y:
            tot = tot + yi
        self.ineq.append(tot - t)

    def linf(self, exprs, name=""):
        t, xs = Expr.lift(exprs[0]), [Expr.lift(e) for e in exprs[1:]]
        for xi in xs:
            self.ineq.append(xi - t)
            self.ineq.append(-xi - t)

    def soc(self, exprs, name=""):
        self.socs.append([Expr.lift(e) for e in exprs])

    def geom(self, exprs, name=""):
        """[t, x1, x2]: geomean(x1, x2) >= t (GEOM, cone.jl:45,161-162; all uses in the reference have two entries:
        ptr.jl:615,667,720, scvx.jl:659, gusto.jl:1129) as the second-order cone |(2 t, x1 - x2)|_2 <= x1 + x2 that
        MathOptInterface's GeoMean -> RSOC -> SOC bridges give ECOS."""
        if len(exprs) != 3:
            raise NotImplementedError("GEOM cone over more than two entries")
        t, x1, x2 = (Expr.lift(e) for e in exprs)
        self.socs.append([x1 + x2, t * 2.0, x1 - x2])

    def sumsq(self, exprs, name="", stage=-2):
        """epigraph of a sum of squares: returns q (a new variable, as Expr) with  sum_i e_i^2 <= q  imposed as the
        rotated second-order cone |(2 e_1, ..., 2 e_n, q - 1)|_2 <= q + 1.  This is how a convex quadratic running cost
        reaches a linear-objective cone solver (JuMP lowers quadratic objectives for ECOS the same way, through its
        quadratic-to-SOC bridge; the minimiser is identical)."""
        q = self._aux(1, stage)[0]
        self.socs.append([q + 1.0] + [Expr.lift(e) * 2.0 for e in exprs] + [q - 1.0])
        self.sq_log[next(iter(q.t))] = [Expr.lift(e) for e in exprs]
        return q

    def add_cost(self, e):
        self.cost = self.cost + Expr.lift(e)

    # compile -----------------------------------------------------------------
    def compile(self):
        """-> dict(A, G patterns (csr, data = entry id), l, soc_dims, W (csr nval x nsrc), offsets, ...).

        Value vector layout: [Avals (nnzA) | Gvals (nnzG) | c (n) | b (p) | h (m)].
        Sign conventions as in the cone solver:  A z = b,  G z + s = h  (G rows: expr <= 0 -> G z <= -const;
        SOC rows: s = expr  ->  -G_expr z + s = const)."""
        n = self.nvar
        soc_rows, q = [], []
        for cone in self.socs:
            q.append(len(cone))
            soc_rows.extend(cone)
        l = len(self.ineq)
        rows_G = list(self.ineq) + soc_rows
        sgnG = [1.0] * l + [-1.0] * len(soc_rows)

        def pattern(rows):
            ind, ptr, coef = [], [0], []
            for e in rows:
                cols = sorted(k for k, v in e.t.items() if not v.is_zero())
                ind.extend(cols)
                coef.extend(e.t[k] for k in cols)
                ptr.append(len(ind))
            return np.array(ptr, dtype=np.int32), np.array(ind, dtype=np.int32), coef

        a_ptr, a_ind, a_coef = pattern(self.eq)
        g_ptr, g_ind, g_coef = pattern(rows_G)
        p, m = len(self.eq), len(rows_G)
        nnzA, nnzG = len(a_ind), len(g_ind)
        # W rows
        wr, wc, wv = [], [], []

        def emit(row, lin, sign=1.0):
            for k, v in lin.t.items():
                if v != 0.0:
                    wr.append(row); wc.append(k); wv.append(sign * v)

        r = 0
        for co in a_coef:
            emit(r, co); r += 1
        gi = 0
        for ri in range(m):
            for _ in range(g_ptr[ri], g_ptr[ri + 1]):
                emit(r, g_coef[gi], sgnG[ri]); r += 1; gi += 1
        off_c = r
        for k, v in self.cost.t.items():
            emit(off_c + k, v)
        r = off_c + n
        off_b = r
        for i, e in enumerate(self.eq):
            emit(off_b + i, e.c, -1.0)
        off_h = off_b + p
        for i, e in enumerate(rows_G):
            emit(off_h + i, e.c, -sgnG[i])
        nval = off_h + m
        W = sp.csr_matrix((wv, (wr, wc)), shape=(nval, self.nsrc))
        W.sum_duplicates(); W.sort_indices()
        A = sp.csr_matrix((np.arange(1, nnzA + 1, dtype=np.float64), a_ind, a_ptr), shape=(p, n))
        G = sp.csr_matrix((np.arange(1, nnzG + 1, dtype=np.float64), g_ind, g_ptr), shape=(m, n))
        return dict(n=n, p=p, m=m, l=l, soc_dims=q, A=A, G=G, W=W, nnzA=nnzA, nnzG=nnzG,
                    off_G=nnzA, off_c=off_c, off_b=off_b, off_h=off_h, nval=nval,
                    cost_const=self.cost.c, var_stage=np.array(self.var_stage, dtype=np.int64))
