"""TEST INFRASTRUCTURE ONLY -- ctypes binding of oracle/_ref/libhiop_ref_harness.so, i.e. the UNMODIFIED
reference CPU path (compiled by oracle/Makefile from /root/reference, driven by oracle/ref_harness.cpp).
Used to (1) pin the numpy/C restatement in kkt_oracle.py, (2) generate tests/golden/*.npz, and (3) as the
"reference" cpu_baseline / --impl reference arm of bench.py. Never imported by the product."""
from __future__ import annotations

import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(_HERE, "_ref", "libhiop_ref_harness.so")
_LIB = None

dp = ctypes.POINTER(ctypes.c_double)
ip = ctypes.POINTER(ctypes.c_int)


def available() -> bool:
    return os.path.exists(SO)


def lib():
    global _LIB
    if _LIB is None:
        L = ctypes.CDLL(SO)
        L.ref_qn_create.restype = ctypes.c_void_p
        L.ref_qn_create.argtypes = [ctypes.c_int] * 4 + [dp] * 4
        L.ref_qn_destroy.argtypes = [ctypes.c_void_p]
        L.ref_qn_sizes.argtypes = [ctypes.c_void_p, ip]
        L.ref_qn_set_iterate.argtypes = [ctypes.c_void_p] + [dp] * 8
        L.ref_qn_set_jac.argtypes = [ctypes.c_void_p, dp, dp]
        L.ref_qn_set_secant.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_double, dp, dp, dp, dp]
        L.ref_qn_update.argtypes = [ctypes.c_void_p, dp, dp, dp, dp]
        L.ref_qn_condense.argtypes = [ctypes.c_void_p, dp, dp]
        L.ref_qn_solve_compressed.argtypes = [ctypes.c_void_p] + [dp] * 7
        L.ref_qn_solve_compressed.restype = ctypes.c_int
        L.ref_qn_hess_solve.argtypes = [ctypes.c_void_p, dp, dp]
        L.ref_qn_hess_times_vec.argtypes = [ctypes.c_void_p, ctypes.c_double, dp, ctypes.c_double, dp, ctypes.c_int]
        L.ref_qn_compute_directions.argtypes = [ctypes.c_void_p, ctypes.POINTER(dp), ctypes.POINTER(dp)]
        L.ref_qn_compute_directions.restype = ctypes.c_int
        L.ref_qn_compute_directions_w_IR.argtypes = [ctypes.c_void_p, ctypes.POINTER(dp), ctypes.POINTER(dp), ctypes.c_double, ctypes.c_int, dp]
        L.ref_qn_compute_directions_w_IR.restype = ctypes.c_int
        L.ref_qn_kkt_full_times_vec.argtypes = [ctypes.c_void_p, ctypes.POINTER(dp), ctypes.POINTER(dp)]
        L.ref_qn_kkt_full_times_vec.restype = ctypes.c_int
        L.ref_qn_hess_update.argtypes = [ctypes.c_void_p, dp, dp, dp, dp, dp, dp, ctypes.POINTER(ctypes.c_int), dp, dp, dp, dp, dp]
        L.ref_qn_hess_update.restype = ctypes.c_int
        L.ref_qn_set_sigma_strategy.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_double]
        L.ref_qn_set_sigma_strategy.restype = None
        L.ref_densekkt_build.argtypes = [ctypes.c_int] * 4 + [dp] * 15 + [ctypes.POINTER(dp), dp]
        L.ref_densekkt_build.restype = ctypes.c_int
        L.ref_qn_lsq_duals.argtypes = [ctypes.c_void_p, dp, dp, dp]
        L.ref_qn_lsq_duals.restype = ctypes.c_int
        L.ref_write_iajaaa.argtypes = [ctypes.c_char_p, ctypes.c_int, ctypes.c_int, dp, ctypes.c_int, ctypes.c_int, ctypes.c_int, dp, dp]
        L.ref_write_iajaaa.restype = ctypes.c_int
        L.ref_qn_residual_update.argtypes = [ctypes.c_void_p, ctypes.POINTER(dp), dp, dp, dp, ctypes.c_double, ctypes.c_double, dp, dp, dp, dp, dp,
                                             ctypes.POINTER(dp), dp]
        L.ref_qn_residual_update.restype = ctypes.c_int
        L.ref_qn_logbar_update.argtypes = [ctypes.c_void_p, ctypes.POINTER(dp), ctypes.c_double, ctypes.c_double, ctypes.c_double, dp, dp, dp, dp]
        L.ref_qn_logbar_update.restype = ctypes.c_int
        L.ref_qn_fraction_to_bdry.argtypes = [ctypes.c_void_p, ctypes.POINTER(dp), ctypes.POINTER(dp), ctypes.c_double, dp, dp]
        L.ref_qn_fraction_to_bdry.restype = ctypes.c_int
        L.ref_qn_adjust_duals.argtypes = [ctypes.c_void_p, ctypes.POINTER(dp), ctypes.c_double, ctypes.c_double, ctypes.POINTER(dp)]
        L.ref_qn_adjust_duals.restype = ctypes.c_int
        L.ref_qn_adjust_small_slacks.argtypes = [ctypes.c_void_p, ctypes.POINTER(dp), ctypes.POINTER(dp), ctypes.c_double, dp, dp, dp, dp,
                                                 ctypes.POINTER(dp)]
        L.ref_qn_adjust_small_slacks.restype = ctypes.c_int
        L.ref_bicgstab_dense.argtypes = [ctypes.c_int, dp, dp, dp, ctypes.c_double, ctypes.c_int, dp]
        L.ref_bicgstab_dense.restype = ctypes.c_int
        L.ref_symdense_factor_solve.argtypes = [ctypes.c_int, dp, ctypes.c_int, dp, dp, dp]
        L.ref_symdense_factor_solve.restype = ctypes.c_int
        L.ref_vec_op.argtypes = [ctypes.c_int, ctypes.c_int, dp, dp, dp, dp, ctypes.c_double, ctypes.c_double]
        L.ref_vec_op.restype = ctypes.c_double
        L.ref_mat_times_vec.argtypes = [ctypes.c_int, ctypes.c_int, dp, ctypes.c_double, dp, ctypes.c_double, dp]
        L.ref_mat_trans_times_vec.argtypes = [ctypes.c_int, ctypes.c_int, dp, ctypes.c_double, dp, ctypes.c_double, dp]
        L.ref_mat_trans_add_to_sym_upper.argtypes = [ctypes.c_int, ctypes.c_int, dp, ctypes.c_int, ctypes.c_int,
                                                     ctypes.c_double, ctypes.c_int, dp]
        L.ref_mat_add_upper_to_sym_upper.argtypes = [ctypes.c_int, dp, ctypes.c_int, ctypes.c_double, ctypes.c_int, dp]
        L.ref_mat_add_sub_diagonal.argtypes = [ctypes.c_int, dp, ctypes.c_int, ctypes.c_double, ctypes.c_int, dp]
        L.ref_sp_add_MDinvMtrans.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ip, ip, dp, ctypes.c_int,
                                             ctypes.c_double, dp, ctypes.c_int, dp]
        L.ref_sp_add_MDinvNtrans.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ip, ip, dp,
                                             ctypes.c_int, ctypes.c_int, ip, ip, dp,
                                             ctypes.c_int, ctypes.c_int, ctypes.c_double, dp, ctypes.c_int, dp]
        _LIB = L
    return _LIB


def _d(a):
    a = np.ascontiguousarray(a, dtype=np.float64)
    return a, a.ctypes.data_as(dp)


def _i(a):
    a = np.ascontiguousarray(a, dtype=np.int32)
    return a, a.ctypes.data_as(ip)


def has_sp_times_vec() -> bool:
    """ref_sp_times_vec is newer than the rest of the harness: an oracle/_ref built before it was added lacks it (make keeps a .so
    that is newer than ref_harness.cpp)"""
    return hasattr(lib(), "ref_sp_times_vec")


def sp_times_vec(trans, m, n, iRow, jCol, vals, y, alpha, x):
    """hiopMatrixSparseTriplet::timesVec (trans = 0) / transTimesVec (trans = 1) with beta = 1 on an m x n triplet matrix; returns y_out"""
    f = lib().ref_sp_times_vec
    f.argtypes = [ctypes.c_int] * 4 + [ip, ip, dp, ctypes.c_double, dp, ctypes.c_double, dp]
    f.restype = None
    (_, pi), (_, pj), (_, pv), (_, px) = _i(iRow), _i(jCol), _d(vals), _d(x)
    y = np.array(y, dtype=np.float64)
    f(trans, m, n, len(iRow), pi, pj, pv, 1.0, y.ctypes.data_as(dp), alpha, px)
    return y


# op codes of ref_vec_op (kept in sync with the enum in ref_harness.cpp)
OPS = dict(axdzpy_w_pattern=1, axzpy=2, axdzpy=3, component_mult=4, component_div=5, component_div_w_sel=6,
           invert=7, select_pattern=8, add_constant=9, add_constant_w_sel=10, scale=11, axpy=12,
           add_logbar_grad=13, add_lin_damping=14, twonorm=20, dot=21, infnorm=22, onenorm=23, logbarrier=24,
           lin_damping_term=25, min_w_pattern=26, frac_to_bdry=27, frac_to_bdry_w_sel=28, sum=29)


def vec_op(op, y, x=None, z=None, sel=None, alpha=0.0, beta=0.0):
    """Runs one hiopVectorPar method; returns (y_out, scalar)."""
    n = y.size
    yy = np.array(y, dtype=np.float64)
    keep = [yy]

    def opt(a):
        if a is None:
            return None
        arr, ptr = _d(a)
        keep.append(arr)
        return ptr

    r = lib().ref_vec_op(OPS[op], n, yy.ctypes.data_as(dp), opt(x), opt(z), opt(sel), alpha, beta)
    return yy, r


class RefQn:
    """One quasi-Newton KKT system replayed through the reference's own classes."""

    def __init__(self, n, m_eq, m_ineq, lmax, ixl, ixu, idl, idu):
        self.n, self.meq, self.mineq, self.lmax = n, m_eq, m_ineq, lmax
        a = [_d(v) for v in (ixl, ixu, idl if m_ineq else np.zeros(1), idu if m_ineq else np.zeros(1))]
        self.h = lib().ref_qn_create(n, m_eq, m_ineq, lmax, *[p for _, p in a])
        sz = (ctypes.c_int * 5)()
        lib().ref_qn_sizes(self.h, sz)
        assert (sz[0], sz[1], sz[2]) == (n, m_eq, m_ineq), list(sz)

    def close(self):
        if self.h:
            lib().ref_qn_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_iterate(self, sxl, sxu, zl, zu, sdl, sdu, vl, vu):
        a = [_d(v) for v in (sxl, sxu, zl, zu, sdl, sdu, vl, vu)]
        lib().ref_qn_set_iterate(self.h, *[p for _, p in a])

    def set_jac(self, Jc, Jd):
        a, pa = _d(Jc)
        b, pb = _d(Jd)
        lib().ref_qn_set_jac(self.h, pa, pb)

    def set_secant(self, sigma, St, Yt, L, D):
        l = St.shape[0]
        a = [_d(v) for v in (St, Yt, L, D)]
        lib().ref_qn_set_secant(self.h, l, float(sigma), *[p for _, p in a])

    def update(self):
        Dx = np.zeros(self.n)
        DhInv = np.zeros(self.n)
        Ddinv = np.zeros(self.mineq)
        t = np.zeros(4)
        lib().ref_qn_update(self.h, Dx.ctypes.data_as(dp), DhInv.ctypes.data_as(dp), Ddinv.ctypes.data_as(dp),
                            t.ctypes.data_as(dp))
        self.t_update = t[0]
        return Dx, DhInv, Ddinv

    def condense(self):
        m = self.meq + self.mineq
        N = np.zeros((m, m))
        t = np.zeros(4)
        lib().ref_qn_condense(self.h, N.ctypes.data_as(dp), t.ctypes.data_as(dp))
        self.t_condense = t[0]
        return N

    def solve_compressed(self, rx, ryc, ryd):
        dx = np.zeros(self.n)
        dyc = np.zeros(self.meq)
        dyd = np.zeros(self.mineq)
        t = np.zeros(4)
        a = [_d(v) for v in (rx, ryc, ryd)]
        rc = lib().ref_qn_solve_compressed(self.h, *[p for _, p in a], dx.ctypes.data_as(dp), dyc.ctypes.data_as(dp),
                                           dyd.ctypes.data_as(dp), t.ctypes.data_as(dp))
        self.t_solve = t[0]
        assert rc == 0
        return dx, dyc, dyd

    def hess_solve(self, rhs):
        x = np.zeros(self.n)
        a, pa = _d(rhs)
        lib().ref_qn_hess_solve(self.h, pa, x.ctypes.data_as(dp))
        return x

    def hess_times_vec(self, beta, y, alpha, x, add_log_term):
        yy = np.array(y, dtype=np.float64)
        a, pa = _d(x)
        lib().ref_qn_hess_times_vec(self.h, beta, yy.ctypes.data_as(dp), alpha, pa, int(add_log_term))
        return yy

    def compute_directions(self, res: dict):
        from .kkt_oracle import RES_NAMES, DIR_NAMES
        sizes = dict(x=self.n, d=self.mineq, yc=self.meq, yd=self.mineq, sxl=self.n, sxu=self.n, sdl=self.mineq,
                     sdu=self.mineq, zl=self.n, zu=self.n, vl=self.mineq, vu=self.mineq)
        rin = [np.ascontiguousarray(res[k], dtype=np.float64) for k in RES_NAMES]
        dout = [np.zeros(sizes[k]) for k in DIR_NAMES]
        RA = (dp * 12)(*[a.ctypes.data_as(dp) for a in rin])
        DA = (dp * 12)(*[a.ctypes.data_as(dp) for a in dout])
        rc = lib().ref_qn_compute_directions(self.h, RA, DA)
        assert rc == 0
        return dict(zip(DIR_NAMES, dout))


    def hess_update(self, x, grad_f, yc, yd, Jc, Jd):
        """hiopHessianLowRank::update -> (l, St[l x n], Yt[l x n], L[l x l], D[l], sigma) after the call."""
        lm = max(self.lmax, 1)
        St, Yt = np.zeros((lm, self.n)), np.zeros((lm, self.n))
        L, D = np.zeros(lm * lm), np.zeros(lm)
        l = ctypes.c_int(0)
        sg = np.zeros(1)
        a = [np.ascontiguousarray(v, dtype=np.float64) for v in (x, grad_f, yc, yd, Jc, Jd)]
        rc = lib().ref_qn_hess_update(self.h, *[v.ctypes.data_as(dp) for v in a], ctypes.byref(l), St.ctypes.data_as(dp), Yt.ctypes.data_as(dp),
                                      L.ctypes.data_as(dp), D.ctypes.data_as(dp), sg.ctypes.data_as(dp))
        assert rc == 0
        ll = l.value
        return ll, St[:ll].copy(), Yt[:ll].copy(), L[:ll * ll].reshape(ll, ll).copy(), D[:ll].copy(), float(sg[0])

    def set_sigma_strategy(self, strategy: int, sigma0: float = 1.0):
        lib().ref_qn_set_sigma_strategy(self.h, int(strategy), ctypes.c_double(sigma0))

    def lsq_duals(self, grad_f):
        """hiopDualsLsqUpdateLinsysRedDenseSymPD::do_lsq_update -> (yc, yd)."""
        g = np.ascontiguousarray(grad_f, dtype=np.float64)
        yc, yd = np.zeros(max(self.meq, 1)), np.zeros(max(self.mineq, 1))
        rc = lib().ref_qn_lsq_duals(self.h, g.ctypes.data_as(dp), yc.ctypes.data_as(dp), yd.ctypes.data_as(dp))
        assert rc == 0
        return yc[:self.meq].copy(), yd[:self.mineq].copy()

    def residual_update(self, itr: dict, c, d, grad, mu, kappa_d, xl, xu, dl, du, crhs):
        """hiopResidual::update -> (residual dict, norms dict)."""
        from .kkt_oracle import RES_NAMES, DIR_NAMES, NORM_NAMES
        sizes = self._sizes()
        keep = [np.ascontiguousarray(itr[k] if np.asarray(itr[k]).size else np.zeros(1), dtype=np.float64) for k in DIR_NAMES]
        IA = (dp * 12)(*[a.ctypes.data_as(dp) for a in keep])
        rout = [np.zeros(max(sizes[k], 1)) for k in DIR_NAMES]
        RA = (dp * 12)(*[a.ctypes.data_as(dp) for a in rout])
        vecs = [np.ascontiguousarray(v if np.asarray(v).size else np.zeros(1), dtype=np.float64) for v in (c, d, grad, xl, xu, dl, du, crhs)]
        nrm = np.zeros(11)
        pv = [v.ctypes.data_as(dp) for v in vecs]
        rc = lib().ref_qn_residual_update(self.h, IA, pv[0], pv[1], pv[2], ctypes.c_double(mu), ctypes.c_double(kappa_d), pv[3], pv[4], pv[5], pv[6],
                                          pv[7], RA, nrm.ctypes.data_as(dp))
        assert rc == 0
        return {rk: rout[i][:sizes[dk]].copy() for i, (rk, dk) in enumerate(zip(RES_NAMES, DIR_NAMES))}, dict(zip(NORM_NAMES, nrm))

    def _blocks(self, d: dict):
        from .kkt_oracle import DIR_NAMES
        keep = [np.ascontiguousarray(d[k] if np.asarray(d[k]).size else np.zeros(1), dtype=np.float64) for k in DIR_NAMES]
        return keep, (dp * 12)(*[a.ctypes.data_as(dp) for a in keep])

    def logbar_update(self, itr: dict, f, mu, kappa_d, grad):
        """hiopLogBarProblem::updateWithNlpInfo -> (f_logbar, grad_x_logbar, grad_d_logbar)."""
        keep, IA = self._blocks(itr)
        g = np.ascontiguousarray(grad, dtype=np.float64)
        gx, gd, fl = np.zeros(self.n), np.zeros(max(self.mineq, 1)), np.zeros(1)
        lib().ref_qn_logbar_update(self.h, IA, ctypes.c_double(f), ctypes.c_double(mu), ctypes.c_double(kappa_d), g.ctypes.data_as(dp),
                                   gx.ctypes.data_as(dp), gd.ctypes.data_as(dp), fl.ctypes.data_as(dp))
        return float(fl[0]), gx, gd[:self.mineq].copy()

    def adjust_duals(self, itr: dict, mu, kappa):
        keep, IA = self._blocks(itr)
        outs = [np.zeros(max(self.n, 1)), np.zeros(max(self.n, 1)), np.zeros(max(self.mineq, 1)), np.zeros(max(self.mineq, 1))]
        OA = (dp * 4)(*[a.ctypes.data_as(dp) for a in outs])
        lib().ref_qn_adjust_duals(self.h, IA, ctypes.c_double(mu), ctypes.c_double(kappa), OA)
        return outs[0][:self.n].copy(), outs[1][:self.n].copy(), outs[2][:self.mineq].copy(), outs[3][:self.mineq].copy()

    def adjust_small_slacks(self, itr: dict, itr_curr: dict, mu, xl, xu, dl, du):
        k1, IA = self._blocks(itr)
        k2, CA = self._blocks(itr_curr)
        b = [np.ascontiguousarray(v if np.asarray(v).size else np.zeros(1), dtype=np.float64) for v in (xl, xu, dl, du)]
        outs = [np.zeros(max(self.n, 1)), np.zeros(max(self.n, 1)), np.zeros(max(self.mineq, 1)), np.zeros(max(self.mineq, 1))]
        OA = (dp * 4)(*[a.ctypes.data_as(dp) for a in outs])
        num = lib().ref_qn_adjust_small_slacks(self.h, IA, CA, ctypes.c_double(mu), *[v.ctypes.data_as(dp) for v in b], OA)
        return num, (outs[0][:self.n].copy(), outs[1][:self.n].copy(), outs[2][:self.mineq].copy(), outs[3][:self.mineq].copy())

    def fraction_to_bdry(self, itr: dict, direction: dict, tau):
        k1, IA = self._blocks(itr)
        k2, DA = self._blocks(direction)
        a = np.zeros(2)
        lib().ref_qn_fraction_to_bdry(self.h, IA, DA, ctypes.c_double(tau), a[:1].ctypes.data_as(dp), a[1:].ctypes.data_as(dp))
        return float(a[0]), float(a[1])

    def _sizes(self):
        return dict(x=self.n, d=self.mineq, yc=self.meq, yd=self.mineq, sxl=self.n, sxu=self.n, sdl=self.mineq,
                    sdu=self.mineq, zl=self.n, zu=self.n, vl=self.mineq, vu=self.mineq)

    def compute_directions_w_ir(self, res: dict, mu: float, maxit: int = 8):
        """hiopKKTLinSys::compute_directions_w_IR -> (directions, (flag, iter, abs_resid, rel_resid))."""
        from .kkt_oracle import RES_NAMES, DIR_NAMES
        sizes = self._sizes()
        rin = [np.ascontiguousarray(res[k], dtype=np.float64) for k in RES_NAMES]
        dout = [np.zeros(sizes[k]) for k in DIR_NAMES]
        RA = (dp * 12)(*[a.ctypes.data_as(dp) for a in rin])
        DA = (dp * 12)(*[a.ctypes.data_as(dp) for a in dout])
        info = np.zeros(4)
        rc = lib().ref_qn_compute_directions_w_IR(self.h, RA, DA, ctypes.c_double(mu), int(maxit), info.ctypes.data_as(dp))
        assert rc == 0
        return dict(zip(DIR_NAMES, dout)), tuple(info)

    def kkt_full_times_vec(self, x: dict):
        from .kkt_oracle import RES_NAMES, DIR_NAMES
        sizes = self._sizes()
        xin = [np.ascontiguousarray(x[k], dtype=np.float64) for k in DIR_NAMES]
        yout = [np.zeros(sizes[k]) for k in DIR_NAMES]
        XA = (dp * 12)(*[a.ctypes.data_as(dp) for a in xin])
        YA = (dp * 12)(*[a.ctypes.data_as(dp) for a in yout])
        rc = lib().ref_qn_kkt_full_times_vec(self.h, XA, YA)
        assert rc == 0
        return dict(zip(RES_NAMES, yout))


def densekkt_build(form, H, Jc, Jd, it, pat, deltas):
    """hiopKKTLinSysDenseXYcYd / XDYcYd::build_kkt_matrix through the reference's own classes. Returns Msys (N x N)."""
    nx, neq, nineq = H.shape[0], Jc.shape[0], Jd.shape[0]
    N = nx + neq + nineq + (nineq if form else 0)
    keep = [np.ascontiguousarray(v, dtype=np.float64) for v in
            (H, Jc if neq else np.zeros(1), Jd if nineq else np.zeros(1), pat["ixl"], pat["ixu"], pat["idl"] if nineq else np.zeros(1),
             pat["idu"] if nineq else np.zeros(1), it["zl"], it["sxl"], it["zu"], it["sxu"], it["vl"] if nineq else np.zeros(1),
             it["sdl"] if nineq else np.zeros(1), it["vu"] if nineq else np.zeros(1), it["sdu"] if nineq else np.zeros(1))]
    dl = [np.ascontiguousarray(d if d.size else np.zeros(1), dtype=np.float64) for d in deltas]
    DA = (dp * 4)(*[a.ctypes.data_as(dp) for a in dl])
    M = np.zeros((N, N))
    n_ret = lib().ref_densekkt_build(form, nx, neq, nineq, *[a.ctypes.data_as(dp) for a in keep], DA, M.ctypes.data_as(dp))
    assert n_ret == N
    return M


def write_iajaaa(directory, counter, M, nx, meq, mineq, rhs, sol):
    """hiopCSR_IO writer -> path of kkt_linsys_<counter>.iajaaa inside `directory`."""
    Ma, pM = _d(M)
    r, pr = _d(rhs)
    x, px = _d(sol)
    rc = lib().ref_write_iajaaa(str(directory).encode(), int(counter), Ma.shape[0], pM, int(nx), int(meq), int(mineq), pr, px)
    assert rc == 0
    return os.path.join(str(directory), f"kkt_linsys_{counter}.iajaaa")


def bicgstab_dense(A, Minv, b, tol, maxit):
    """hiopBiCGStabSolver::solve on a dense system with a dense left preconditioner. Returns (x, (flag, iter, abs, rel))."""
    n = b.size
    Aa, pA = _d(A)
    Ma, pM = _d(Minv)
    x = np.array(b, dtype=np.float64).copy()
    info = np.zeros(4)
    lib().ref_bicgstab_dense(n, pA, pM, x.ctypes.data_as(dp), ctypes.c_double(tol), int(maxit), info.ctypes.data_as(dp))
    return x, tuple(info)


def symdense_factor_solve(M_upper, rhs=None):
    """hiopLinSolverSymDenseLapack::matrixChanged (+ solve). Returns (ret, solution or None, factor, times)."""
    N = M_upper.shape[0]
    M, pM = _d(M_upper)
    fac = np.zeros((N, N))
    t = np.zeros(2)
    if rhs is None:
        x = np.zeros(max(N, 1))
        nrhs = 0
    else:
        x = np.array(rhs, dtype=np.float64).reshape(-1, N).copy()
        nrhs = x.shape[0]
    ret = lib().ref_symdense_factor_solve(N, pM, nrhs, x.ctypes.data_as(dp), fac.ctypes.data_as(dp), t.ctypes.data_as(dp))
    sol = None if rhs is None else x.reshape(np.shape(rhs))
    return ret, sol, fac, t
