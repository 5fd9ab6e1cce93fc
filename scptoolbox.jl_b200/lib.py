"""ctypes binding of libscpb.so -- the C ABI declared in include/scpb.h.

This is the only way the Python host reaches the GPU path: there is no CPU fallback.
If the shared library is missing, or no CUDA device is present when a handle is created,
the call raises -- loudly -- instead of computing anything on the host.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.environ.get("SCPB_LIBRARY") or os.path.join(HERE, "libscpb.so")   # override: A/B runs of kernel variants

MODEL_DBLINT, MODEL_ROCKET, MODEL_STARSHIP, MODEL_QUADROTOR, MODEL_FREEFLYER, MODEL_RENDEZVOUS2D = 1, 2, 3, 4, 5, 6
MODEL_OSCILLATOR = 7
FOH, IMPULSE = 0, 1

_lib = None

_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int32)

# name -> (restype, argtypes); must list EVERY symbol include/scpb.h declares
SIGNATURES = {
    "scpb_create": (C.c_int32, [C.c_int32, C.POINTER(C.c_void_p)]),
    "scpb_destroy": (C.c_int32, [C.c_void_p]),
    "scpb_last_error": (C.c_int32, [C.c_void_p, C.c_char_p, C.c_size_t]),
    "scpb_version": (C.c_int32, []),
    "scpb_launch_count": (C.c_int64, [C.c_void_p]),
    "scpb_stream": (C.c_void_p, [C.c_void_p]),
    "scpb_sync": (C.c_int32, [C.c_void_p]),
    "scpb_model_set": (C.c_int32, [C.c_void_p, C.c_int32, _dp, C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "scpb_discretize": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                    _dp, _dp, _dp, _dp, _dp, C.c_double,
                                    _dp, _dp, _dp, _dp, _dp, _dp, _dp, _ip, _dp]),
    "scpb_discretize_dev": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_void_p]),
    "scpb_propagate": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _dp, _dp, _dp, _dp, _dp, _dp]),
    "scpb_cone_setup": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, _ip, _ip, _ip, _ip, C.c_int32,
                                    C.c_int32, _ip, _ip, C.POINTER(C.c_void_p)]),
    "scpb_order_rcm": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, _ip, _ip, _ip, _ip, C.c_int32, C.c_int32, _ip, _ip]),
    "scpb_cone_info": (C.c_int32, [C.c_void_p, C.POINTER(C.c_int64)]),
    "scpb_cone_free": (C.c_int32, [C.c_void_p]),
    "scpb_cone_solve": (C.c_int32, [C.c_void_p, C.c_int32, _dp, _dp, _dp, _dp, _dp, C.c_void_p,
                                    _dp, _dp, _dp, _dp, _dp, _dp, _ip, _ip, _dp]),
    "scpb_ptr_setup": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, _ip, _ip, _dp, _dp, _dp, C.POINTER(C.c_void_p)]),
    "scpb_ptr_free": (C.c_int32, [C.c_void_p]),
    "scpb_ptr_set_par": (C.c_int32, [C.c_void_p, _dp, C.c_int32]),
    "scpb_ptr_set_homotopy": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int32, _dp, C.c_double]),
    "scpb_ptr_set_homotopy_beta": (C.c_int32, [C.c_void_p, C.c_int32, _dp]),
    "scpb_ptr_homotopy_result": (C.c_int32, [C.c_void_p, C.c_int32, _ip, _ip, C.c_int32, _ip, _dp]),
    "scpb_ptr_solve": (C.c_int32, [C.c_void_p, C.c_int32, _dp, _dp, _dp, C.c_void_p, _dp, _dp, _dp, _ip, _ip,
                                   _dp, _dp, _ip, _dp]),
    "scpb_scvx_attach": (C.c_int32, [C.c_void_p, C.c_void_p, _ip, _ip, _dp, _dp]),
    "scpb_gusto_attach": (C.c_int32, [C.c_void_p, C.c_void_p, _ip, _ip, _dp, _dp, _dp]),
    "scpb_gusto_solve": (C.c_int32, [C.c_void_p, C.c_int32, _dp, _dp, _dp, C.c_void_p, _dp, _dp, _dp, _ip, _ip,
                                     _dp, _dp, _ip, _dp, _dp, _dp]),
    "scpb_scvx_solve": (C.c_int32, [C.c_void_p, C.c_int32, _dp, _dp, _dp, C.c_void_p, _dp, _dp, _dp, _ip, _ip,
                                    _dp, _dp, _ip, _dp, _dp]),
    "scpb_debug_ipm_trace": (C.c_int32, [C.c_void_p, _dp, C.c_int32]),
    "scpb_debug_level_profile": (C.c_int32, [C.c_void_p, C.POINTER(C.c_int64), C.c_int32]),
    "scpb_debug_kkt_solve": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, _ip, _ip, _ip, _ip, C.c_int32, C.c_int32,
                                         _ip, _ip, _dp, _dp, _dp, C.c_double, C.c_double, _dp, _dp, C.POINTER(C.c_int64)]),
    "scpb_debug_kkt_solve_sn": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, _ip, _ip, _ip, _ip, C.c_int32, C.c_int32,
                                         _ip, _ip, _dp, _dp, _dp, C.c_double, C.c_double, _dp, _dp, C.POINTER(C.c_int64)]),
    "scpb_debug_kkt_solve_hy": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, _ip, _ip, _ip, _ip, C.c_int32, C.c_int32,
                                         _ip, _ip, _dp, _dp, _dp, C.c_double, C.c_double, C.c_int32, _dp, _dp,
                                         C.POINTER(C.c_int64)]),
    "scpb_debug_fp64_peak": (C.c_int32, [C.c_void_p, _dp]),
    "scpb_debug_constraints": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _dp, _dp, _dp, _dp,
                                           _dp, _dp, _dp, _dp]),
    "scpb_debug_kkt_solve_dev": (C.c_int32, [C.c_void_p, C.c_int32, _dp, _dp, _dp, C.c_double, _dp, _dp, _ip]),
    "scpb_debug_kkt_new": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, _ip, _ip, _ip, _ip, C.c_int32, C.c_int32, _ip, _ip,
                                       C.POINTER(C.c_void_p), C.POINTER(C.c_int64)]),
    "scpb_debug_kkt_factor": (C.c_int32, [C.c_void_p, _dp, _dp, _dp, C.c_double, C.c_double, C.c_double, C.c_double, _dp]),
    "scpb_debug_kkt_resolve": (C.c_int32, [C.c_void_p, _dp, _dp]),
    "scpb_debug_kkt_free": (C.c_int32, [C.c_void_p]),
}


class ConeOpts(C.Structure):
    _fields_ = [("feastol", C.c_double), ("abstol", C.c_double), ("reltol", C.c_double),
                ("delta", C.c_double), ("delta_dyn", C.c_double), ("maxit", C.c_int32), ("nref", C.c_int32),
                ("verbose", C.c_int32), ("group", C.c_int32), ("equil", C.c_int32), ("threads", C.c_int32), ("lanes", C.c_int32)]


class PtrDesc(C.Structure):
    _fields_ = [(k, C.c_int32) for k in
                ("N", "Nsub", "nx", "nu", "np", "ns", "nf", "nsrc", "oA", "oBm", "oBp", "oF", "or_", "oE", "oC", "oD",
                 "oG", "ors", "oxh", "ouh", "oph", "nval", "vx", "vu", "vp", "q_exit", "iter_max", "ng")] + \
               [(k, C.c_double) for k in ("eps_abs", "eps_rel", "feas_tol")] + \
               [("method", C.c_int32)]       # FOH / IMPULSE; appended last, so a zero-initialised descriptor means FOH


class ScvxDesc(C.Structure):        # scpb_scvx_desc (include/scpb.h)
    _fields_ = [(k, C.c_double) for k in ("lam", "rho_0", "rho_1", "rho_2", "beta_sh", "beta_gr", "eta_init", "eta_lb",
                                           "eta_ub")] + [(k, C.c_int32) for k in ("oeta", "n_ic", "n_tc", "reserved")]


class GustoDesc(C.Structure):       # scpb_gusto_desc (include/scpb.h)
    _fields_ = [(k, C.c_double) for k in ("lam_init", "lam_max", "rho_0", "rho_1", "beta_sh", "beta_gr", "gamma_fail",
                                           "eta_init", "eta_lb", "eta_ub", "mu")] + \
               [(k, C.c_int32) for k in ("iter_mu", "q_tr", "oeta", "olam", "nsq", "reserved")]


CONE_STATUS = {0: "OPTIMAL", 1: "ITERATION_LIMIT", 2: "NUMERICAL_ERROR", 3: "ALMOST_OPTIMAL", 4: "INFEASIBLE",
               5: "DUAL_INFEASIBLE"}


class ScpbError(RuntimeError):
    pass


def load():
    """dlopen libscpb.so and bind every exported symbol; raises if the library is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(SO):
            raise ScpbError(f"{SO} not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                            "(there is no CPU fallback)")
        lib = C.CDLL(SO)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def _f64(a):
    a = np.ascontiguousarray(a, dtype=np.float64)
    return a, a.ctypes.data_as(_dp)


class Handle:
    """Opaque library handle bound to one CUDA device + stream (include/scpb.h)."""

    def __init__(self, device: int = 0):
        self.lib = load()
        h = C.c_void_p()
        rc = self.lib.scpb_create(device, C.byref(h))
        if rc != 0 or not h.value:
            raise ScpbError(f"scpb_create(device={device}) failed with status {rc}: no usable CUDA device "
                            "(the product path has no CPU fallback)")
        self.h = h
        self.nx = self.nu = self.np = 0
        self.model_id = 0

    def close(self):
        if getattr(self, "h", None) is not None and self.h.value:
            self.lib.scpb_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int, what: str):
        if rc != 0:
            buf = C.create_string_buffer(512)
            self.lib.scpb_last_error(self.h, buf, 512)
            raise ScpbError(f"{what} failed ({rc}): {buf.value.decode(errors='replace')}")

    @property
    def launches(self) -> int:
        return int(self.lib.scpb_launch_count(self.h))

    @property
    def stream(self) -> int:
        return int(self.lib.scpb_stream(self.h) or 0)

    def sync(self):
        self._check(self.lib.scpb_sync(self.h), "scpb_sync")

    def model_set(self, model_id: int, par, nx: int, nu: int, np_: int):
        par, pp = _f64(par)
        self._check(self.lib.scpb_model_set(self.h, model_id, pp, par.size, nx, nu, np_), "scpb_model_set")
        self.model_id, self.nx, self.nu, self.np = model_id, nx, nu, np_

    def discretize(self, t_grid, xd, ud, p, iSx_diag, feas_tol, Nsub, method=FOH):
        """discretize! for a batch: xd (B, N, nx), ud (B, N, nu), p (B, np) host arrays.

        Returns a dict of Julia-layout arrays A (B, N-1, nx*nx) ..., feas (B,), seconds.
        """
        xd, pxd = _f64(xd)
        ud, pud = _f64(ud)
        p, pp = _f64(p)
        tg, ptg = _f64(t_grid)
        iS, piS = _f64(iSx_diag)
        B, N = xd.shape[0], xd.shape[1]
        nx, nu, np_ = self.nx, self.nu, self.np
        assert xd.shape == (B, N, nx) and ud.shape == (B, N, nu) and p.shape == (B, np_), \
            (xd.shape, ud.shape, p.shape)
        M = N - 1
        out = dict(A=np.empty((B, M, nx * nx)), Bm=np.empty((B, M, nx * nu)), Bp=np.empty((B, M, nx * nu)),
                   F=np.empty((B, M, nx * np_)), r=np.empty((B, M, nx)), E=np.empty((B, M, nx * nx)),
                   defect=np.empty((B, M, nx)), feas=np.zeros(B, dtype=np.int32))
        sec = C.c_double(0.0)
        g = lambda k: out[k].ctypes.data_as(_dp)
        rc = self.lib.scpb_discretize(self.h, method, B, N, Nsub, ptg, pxd, pud, pp, piS, float(feas_tol),
                                      g("A"), g("Bm"), g("Bp"), g("F"), g("r"), g("E"), g("defect"),
                                      out["feas"].ctypes.data_as(_ip), C.byref(sec))
        self._check(rc, "scpb_discretize")
        out["seconds"] = sec.value
        return out

    def propagate(self, t_grid, xd, ud, p, res, method=FOH):
        """propagate(sol, pbm; res) for a batch (discretization.jl:515-562): xd (B, N, nx), ud (B, N, nu), p (B, np).

        Returns (tc (res,), xc (B, res, nx), seconds): per seed xc[b].T is the reference's nx x res matrix."""
        xd, pxd = _f64(xd)
        ud, pud = _f64(ud)
        p, pp = _f64(p)
        tg, ptg = _f64(t_grid)
        B, N = xd.shape[0], xd.shape[1]
        assert xd.shape == (B, N, self.nx) and ud.shape == (B, N, self.nu) and p.shape == (B, self.np)
        if method == IMPULSE:     # discretization.jl:539-558: xd[:,1] + ceil(res/(N-1)) columns per interval
            sub = -(-int(res) // (N - 1))
            ncol = 1 + (N - 1) * sub
        else:
            ncol = int(res)
        xc = np.empty((B, ncol, self.nx))
        sec = C.c_double(0.0)
        rc = self.lib.scpb_propagate(self.h, method, B, N, int(res), ptg, pxd, pud, pp, xc.ctypes.data_as(_dp),
                                     C.byref(sec))
        self._check(rc, "scpb_propagate")
        if method == IMPULSE:
            dt = float(np.sqrt(np.finfo(float).eps))          # the reference's tiny "impulse duration" offset
            tc = [0.0]
            for k in range(N - 1):
                seg = [(1.0 - j / (sub - 1)) * tg[k] + (j / (sub - 1)) * tg[k + 1] for j in range(sub)]
                seg[0] += dt
                tc.extend(seg)
            return np.array(tc), xc, sec.value
        d = res - 1
        tc = np.array([(1.0 - j / d) * 0.0 + (j / d) * 1.0 for j in range(res)])
        return tc, xc, sec.value

    def fp64_peak(self):
        """Measured fp64 FMA throughput of this device in TFLOP/s (scpb_debug_fp64_peak)."""
        v = C.c_double(0.0)
        self._check(self.lib.scpb_debug_fp64_peak(self.h, C.byref(v)), "scpb_debug_fp64_peak")
        return v.value

    def debug_constraints(self, t_grid, xd, ud, p, ns, ng):
        """Test hook (scpb_debug_constraints): the selected model's constraint pack at every seed and node.
        Returns s (B, N, ns), C (B, N, ns, nx), D (B, N, ns, nu), G (B, N, ns, ng)."""
        xd, pxd = _f64(xd)
        ud, pud = _f64(ud)
        p, pp = _f64(p)
        tg, ptg = _f64(t_grid)
        B, N = xd.shape[0], xd.shape[1]
        assert xd.shape == (B, N, self.nx) and ud.shape == (B, N, self.nu) and p.shape == (B, self.np)
        out = dict(s=np.empty((B, N, ns)), C=np.empty((B, N, ns, self.nx)), D=np.empty((B, N, ns, self.nu)),
                   G=np.empty((B, N, ns, ng)))
        g = lambda k: out[k].ctypes.data_as(_dp)
        rc = self.lib.scpb_debug_constraints(self.h, B, N, ns, ng, ptg, pxd, pud, pp, g("s"), g("C"), g("D"), g("G"))
        self._check(rc, "scpb_debug_constraints")
        return out

    def discretize_dev(self, t_grid, xd, ud, p, iSx_diag, feas_tol, Nsub, A, Bm, Bp, F, r, E, defect, feas,
                       B, N, method=FOH):
        """Device-pointer variant; every array argument is an integer device address."""
        rc = self.lib.scpb_discretize_dev(self.h, method, B, N, Nsub, t_grid, xd, ud, p, iSx_diag,
                                          float(feas_tol), A, Bm, Bp, F, r, E, defect, feas)
        self._check(rc, "scpb_discretize_dev")


def _i32(a):
    a = np.ascontiguousarray(a, dtype=np.int32)
    return a, a.ctypes.data_as(_ip)


class ConeProblem:
    """Pattern-shared batched cone program (scpb_cone_*).  A, G: scipy CSR patterns (values ignored)."""

    def __init__(self, handle: "Handle", A, G, l: int, soc_dims=(), perm=None):
        self.hd = handle
        self.lib = handle.lib
        self.n, self.p, self.m = A.shape[1], A.shape[0], G.shape[0]
        A = A.tocsr(); G = G.tocsr()
        A.sort_indices(); G.sort_indices()
        self.nnzA, self.nnzG = A.nnz, G.nnz
        self._keep = [_i32(A.indptr), _i32(A.indices), _i32(G.indptr), _i32(G.indices), _i32(list(soc_dims) or [0])]
        pp = None
        if perm is not None:
            self._keep.append(_i32(perm))
            pp = self._keep[-1][1]
        c = C.c_void_p()
        k = self._keep
        rc = self.lib.scpb_cone_setup(handle.h, self.n, self.p, self.m, k[0][1], k[1][1], k[2][1], k[3][1],
                                      int(l), len(soc_dims), k[4][1], pp, C.byref(c))
        handle._check(rc, "scpb_cone_setup")
        self.c = c
        self.l, self.soc_dims = int(l), list(soc_dims)

    def info(self):
        buf = (C.c_int64 * 24)()
        self.lib.scpb_cone_info(self.c, buf)
        keys = ["nk", "nnzL", "levels", "factor_ops", "assembly_ops", "nwm", "group", "capacity"]
        d = dict(zip(keys, [int(v) for v in buf[:8]]))
        d["cycles"] = dict(zip(["equilibrate", "start_point", "residuals", "scale_assemble", "factor", "kkt_solves",
                                "linesearch_update", "total", "ldl_forward", "ldl_backward", "ldl_count",
                                "factor_count"], [int(v) for v in buf[8:20]]))
        d["hybrid"] = dict(zip(["cut_used", "levels", "top_levels", "cut_built"], [int(v) for v in buf[20:24]]))
        fc = d["cycles"]["factor_count"]
        d["cycles"]["factor_count"] = fc & 0xffffffff      # interior-point iterations of CTA 0
        d["cycles"]["factor_retries"] = fc >> 32           # factorisations repeated with a larger static regularisation
        return d

    def ipm_trace(self, rows=256):
        """rows of the SCPB_IPM_TRACE diagnostic (see include/scpb.h); empty when tracing is off"""
        buf = np.zeros((rows, 10))
        n = self.lib.scpb_debug_ipm_trace(self.c, buf.ctypes.data_as(_dp), rows)
        if n <= 0:
            return buf[:0]
        buf = buf[:n]
        return buf[(buf[:, 0] > 0) | (np.arange(n) == 0)]

    def level_profile(self):
        """(3, levels) cycle counters [factor, forward, backward] of CTA 0 (needs SCPB_LEVEL_PROFILE=1)."""
        nl = self.info()["levels"]
        buf = (C.c_int64 * (3 * nl))()
        rc = self.lib.scpb_debug_level_profile(self.c, buf, 3 * nl)
        if rc != 0:
            raise ScpbError(f"scpb_debug_level_profile failed ({rc})")
        return np.array(buf[:], dtype=np.int64).reshape(3, nl)

    def close(self):
        if getattr(self, "c", None) is not None and self.c.value:
            self.lib.scpb_cone_free(self.c)
            self.c = C.c_void_p()

    def debug_kkt_solve_dev(self, Avals, Gvals, wm, delta, rhs):
        """Test hook: one reduced-KKT assemble + factor + solve on the device for a batch (see include/scpb.h)."""
        Avals, pA = _f64(Avals); Gvals, pG = _f64(Gvals); wm, pw = _f64(wm); rhs, pr = _f64(rhs)
        B = rhs.shape[0]
        assert rhs.shape == (B, self.n + self.p)
        sol = np.zeros_like(rhs)
        bad = np.zeros(B, dtype=np.int32)
        rc = self.lib.scpb_debug_kkt_solve_dev(self.c, B, pA, pG, pw, float(delta), pr, sol.ctypes.data_as(_dp),
                                               bad.ctypes.data_as(_ip))
        self.hd._check(rc, "scpb_debug_kkt_solve_dev")
        return sol, bad

    def solve(self, Avals, Gvals, c, b, h, **opts):
        """Batched solve; arrays are (B, nnzA), (B, nnzG), (B, n), (B, p), (B, m)."""
        Avals, pA = _f64(Avals); Gvals, pG = _f64(Gvals)
        c, pc = _f64(c); b, pb = _f64(b); h, ph = _f64(h)
        B = c.shape[0]
        assert Avals.shape == (B, self.nnzA) and Gvals.shape == (B, self.nnzG), (Avals.shape, Gvals.shape)
        assert c.shape == (B, self.n) and b.shape == (B, self.p) and h.shape == (B, self.m)
        o = ConeOpts()
        o.nref = -1
        o.equil = -1
        for k_, v in opts.items():
            setattr(o, k_, v)
        out = dict(x=np.empty((B, self.n)), y=np.empty((B, self.p)), z=np.empty((B, self.m)),
                   s=np.empty((B, self.m)), pobj=np.empty(B), dobj=np.empty(B),
                   status=np.zeros(B, dtype=np.int32), iters=np.zeros(B, dtype=np.int32))
        sec = C.c_double(0.0)
        g = lambda k_: out[k_].ctypes.data_as(_dp)
        rc = self.lib.scpb_cone_solve(self.c, B, pA, pG, pc, pb, ph, C.cast(C.byref(o), C.c_void_p), g("x"), g("y"),
                                      g("z"), g("s"), g("pobj"), g("dobj"), out["status"].ctypes.data_as(_ip),
                                      out["iters"].ctypes.data_as(_ip), C.byref(sec))
        self.hd._check(rc, "scpb_cone_solve")
        out["seconds"] = sec.value
        return out


def debug_kkt_solve(A, G, l, soc_dims, perm, Avals, Gvals, wm, delta, rhs, delta_dyn=0.0, supernodal=False, hybrid_cut=0):
    """CPU interpreter of the index programs for one seed (test hook, see include/scpb.h); supernodal=True runs the
    dense-panel program instead of the scalar level-scheduled one, hybrid_cut > 0 the hybrid program (scalar below that
    supernodal level, in-place panels above)."""
    lib = load()
    A = A.tocsr(); G = G.tocsr(); A.sort_indices(); G.sort_indices()
    n, p, m = A.shape[1], A.shape[0], G.shape[0]
    a0, a1, g0, g1 = _i32(A.indptr), _i32(A.indices), _i32(G.indptr), _i32(G.indices)
    sd = _i32(list(soc_dims) or [0])
    pm = _i32(perm) if perm is not None else (None, None)
    Av, pAv = _f64(Avals); Gv, pGv = _f64(Gvals); wmv, pwm = _f64(wm); r, pr = _f64(rhs)
    sol = np.zeros(n + p)
    info = (C.c_int64 * 8)()
    if hybrid_cut > 0:
        rc = lib.scpb_debug_kkt_solve_hy(n, p, m, a0[1], a1[1], g0[1], g1[1], int(l), len(soc_dims), sd[1], pm[1],
                                         pAv, pGv, pwm, float(delta), float(delta_dyn), int(hybrid_cut), pr,
                                         sol.ctypes.data_as(_dp), info)
        if rc != 0:
            raise ScpbError(f"scpb_debug_kkt_solve_hy failed ({rc})")
        keys = ("levels", "top_levels", "top_supernodes", "top_columns", "bridge_factor_items", "bridge_factor_ops",
                "bridge_forward_items", "scalar_levels")
        return sol, dict(zip(keys, [int(v) for v in info]))
    if supernodal:
        rc = lib.scpb_debug_kkt_solve_sn(n, p, m, a0[1], a1[1], g0[1], g1[1], int(l), len(soc_dims), sd[1], pm[1],
                                         pAv, pGv, pwm, float(delta), float(delta_dyn), pr, sol.ctypes.data_as(_dp), info)
        if rc != 0:
            raise ScpbError(f"scpb_debug_kkt_solve_sn failed ({rc})")
        keys = ("supernodes", "sn_levels", "panel_doubles", "update_entries", "max_width", "max_rows", "levels", "nnzL")
        return sol, dict(zip(keys, [int(v) for v in info]))
    rc = lib.scpb_debug_kkt_solve(n, p, m, a0[1], a1[1], g0[1], g1[1], int(l), len(soc_dims), sd[1], pm[1],
                                  pAv, pGv, pwm, float(delta), float(delta_dyn), pr, sol.ctypes.data_as(_dp), info)
    if rc != 0:
        raise ScpbError(f"scpb_debug_kkt_solve failed ({rc})")
    return sol, dict(nnzL=int(info[0]), levels=int(info[1]), factor_ops=int(info[2]), assembly_ops=int(info[3]),
                     split_items=int(info[4]))
