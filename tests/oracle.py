"""Loader for the CPU oracle (oracle/taylor_oracle.c) — TEST INFRASTRUCTURE.

Only tests/, __graft_entry__.smoke() and bench.py's CPU legs import this. The library is built by
oracle/Makefile into oracle/_build/ (two ISA levels; the one matching the host CPU is loaded). If the
prebuilt library is missing it is built on the spot with gcc (a one-second compile).
"""
import ctypes as C
import os
import subprocess
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")

PAIRWISE = 1  # default-mode (non-compact) summation order of the reference
FMA = 2       # sequential + fused multiply-add: the order the CUDA kernels use
SEQ = 0       # compact-mode summation order, no contraction
SCALAR_TAIL = 4  # width 4 / 8 only: step size and state update lane by lane instead of on SIMD vectors (A/B check)

_dp = C.POINTER(C.c_double)


def _cpu_has_avx512():
    try:
        with open("/proc/cpuinfo") as f:
            for line in f:
                if line.startswith("flags"):
                    fl = line.split()
                    return all(x in fl for x in ("avx512f", "avx512dq", "avx512bw", "avx512vl", "avx512cd"))
    except OSError:
        pass
    return False


def isa_level():
    return "v4" if _cpu_has_avx512() else "v3"


def _load():
    path = os.path.join(ORACLE_DIR, "_build", "liboracle_%s.so" % isa_level())
    src = os.path.join(ORACLE_DIR, "taylor_oracle.c")
    if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(src):
        subprocess.run(["make", "-C", ORACLE_DIR], check=True, capture_output=True)
    return C.CDLL(path)


lib = _load()


def _desc_ptr(program):
    return C.byref(program.desc)


def _arr(a):
    return a.ctypes.data_as(_dp)


def jet(program, state, pars=None, t_hi=None, lane=0, mode=FMA):
    """Full tape of one lane: array [order + 1, n_uvars]."""
    P = program
    state = np.ascontiguousarray(state, dtype=np.float64).reshape(P.n_eq, -1)
    batch = state.shape[1]
    pars = np.zeros((max(P.n_pars, 1), batch)) if pars is None else np.ascontiguousarray(pars, dtype=np.float64)
    t_hi = np.zeros(batch) if t_hi is None else np.ascontiguousarray(t_hi, dtype=np.float64)
    out = np.empty((P.order + 1, P.n_uvars))
    rc = lib.oracle_jet_w1(_desc_ptr(P), C.c_uint32(batch), _arr(state), _arr(pars), _arr(t_hi), C.c_uint32(lane),
                           _arr(out), C.c_int(mode))
    assert rc == 0
    return out


class OracleIntegrator:
    """CPU restatement of taylor_adaptive_batch<double>: same arrays, same semantics, lock-step lanes."""

    def __init__(self, program, state, batch, pars=None, time=0.0, mode=FMA, width=1):
        P = self.P = program
        self.n = batch
        self.mode = mode
        self.w = width
        self.state = np.array(state, dtype=np.float64).reshape(P.n_eq, batch).copy()
        self.pars = np.zeros((max(P.n_pars, 1), batch)) if pars is None else \
            np.array(pars, dtype=np.float64).reshape(P.n_pars, batch).copy()
        self.t_hi = np.broadcast_to(np.asarray(time, dtype=np.float64), (batch,)).copy()
        self.t_lo = np.zeros(batch)
        self.last_h = np.zeros(batch)
        self.tc = np.zeros((P.n_eq, P.order + 1, batch))
        self.step_outcome = np.zeros(batch, dtype=np.int64)
        self.prop_outcome = np.zeros(batch, dtype=np.int64)
        self.min_h = np.zeros(batch)
        self.max_h = np.zeros(batch)
        self.n_steps = np.zeros(batch, dtype=np.uint64)

    def _fn(self, name):
        return getattr(lib, "%s_w%d" % (name, self.w))

    def step(self, max_delta_t=None, backward=False, write_tc=False, lanes=None):
        n = self.n
        if max_delta_t is None:
            max_delta_t = np.full(n, -np.inf if backward else np.inf)
        mdt = np.ascontiguousarray(np.broadcast_to(max_delta_t, (n,)), dtype=np.float64)
        b, e = lanes if lanes is not None else (0, n)
        rc = self._fn("oracle_step_full")(
            _desc_ptr(self.P), C.c_uint32(n), C.c_uint32(b), C.c_uint32(e), _arr(self.state), _arr(self.pars),
            _arr(self.t_hi), _arr(self.t_lo), _arr(mdt), _arr(self.last_h),
            self.step_outcome.ctypes.data_as(C.POINTER(C.c_int64)), _arr(self.tc) if write_tc else None,
            C.c_int(self.mode))
        assert rc == 0

    def propagate_until(self, t_hi, t_lo=None, max_delta_t=None, max_steps=0, write_tc=False, lockstep=True,
                        n_threads=1):
        n = self.n
        th = np.ascontiguousarray(np.broadcast_to(t_hi, (n,)), dtype=np.float64)
        tl = None if t_lo is None else np.ascontiguousarray(np.broadcast_to(t_lo, (n,)), dtype=np.float64)
        md = None if max_delta_t is None else np.ascontiguousarray(np.broadcast_to(max_delta_t, (n,)), dtype=np.float64)
        fn = self._fn("oracle_propagate_until")

        def run(b, e):
            rc = fn(_desc_ptr(self.P), C.c_uint32(n), C.c_uint32(b), C.c_uint32(e), _arr(self.state), _arr(self.pars),
                    _arr(self.t_hi), _arr(self.t_lo), _arr(th), None if tl is None else _arr(tl),
                    None if md is None else _arr(md), C.c_uint64(max_steps), _arr(self.last_h),
                    self.prop_outcome.ctypes.data_as(C.POINTER(C.c_int64)), _arr(self.min_h), _arr(self.max_h),
                    self.n_steps.ctypes.data_as(C.POINTER(C.c_uint64)), _arr(self.tc) if write_tc else None,
                    C.c_int(self.mode), C.c_int(1 if lockstep else 0))
            assert rc == 0

        if n_threads <= 1 or lockstep:
            run(0, n)
        else:
            # Disjoint lane ranges (multiples of the vector width) on a thread pool; ctypes drops the GIL.
            w = max(self.w, 1)
            per = -(-n // n_threads)
            per = -(-per // w) * w
            ranges = [(b, min(b + per, n)) for b in range(0, n, per)]
            with ThreadPoolExecutor(max_workers=n_threads) as ex:
                list(ex.map(lambda r: run(*r), ranges))

    def d_output(self, tau):
        tau = np.ascontiguousarray(np.broadcast_to(tau, (self.n,)), dtype=np.float64)
        out = np.empty((self.P.n_eq, self.n))
        rc = lib.oracle_d_output_w1(_desc_ptr(self.P), C.c_uint32(self.n), _arr(self.tc), _arr(tau), _arr(out))
        assert rc == 0
        return out

    def propagate_grid(self, grid, max_delta_t=None, max_steps=0):
        """propagate_grid_impl(), src/taylor_adaptive_batch.cpp:1545-2055, restated with the oracle's step() and
        dense output (argument checks left to the product's tests). grid: [n_pts, batch]. Returns [n_pts, n_eq, batch]."""
        import heyoka_b200 as hb
        n, n_eq = self.n, self.P.n_eq
        grid = np.asarray(grid, dtype=np.float64).reshape(-1, n)
        n_pts = grid.shape[0]
        mdt = np.full(n, np.inf) if max_delta_t is None else np.broadcast_to(np.asarray(max_delta_t, float), (n,))
        ret = np.full((n_pts, n_eq, n), np.nan)
        TL, SUCCESS, NF, STEP_LIMIT = (hb.taylor_outcome.time_limit, hb.taylor_outcome.success,
                                       hb.taylor_outcome.err_nf_state, hb.taylor_outcome.step_limit)

        def dsub(ahi, alo, bhi, blo):  # dfloat a - b (include/heyoka/detail/dfloat.hpp:157-186)
            return hb._dfloat_add(np.atleast_1d(ahi), np.atleast_1d(alo), -np.atleast_1d(bhi), -np.atleast_1d(blo))

        def dlt(ahi, alo, bhi, blo):
            return (ahi < bhi) | ((ahi == bhi) & (alo < blo))

        # :1697-1722
        self.propagate_until(grid[0], max_delta_t=None if max_delta_t is None else mdt, max_steps=max_steps,
                             write_tc=True)
        if np.any(self.prop_outcome != TL):
            self.min_h[:] = np.inf
            self.max_h[:] = 0
            self.n_steps[:] = 0
            return ret
        ret[0] = self.state
        rem_hi, rem_lo = dsub(grid[-1], np.zeros(n), self.t_hi, self.t_lo)  # :1728-1739
        t_dir = (rem_hi > 0) | ((rem_hi == 0) & (rem_lo >= 0))
        self.n_steps[:] = 0
        self.min_h[:] = np.inf
        self.max_h[:] = 0
        cur = np.ones(n, dtype=np.int64)
        it = 0
        while np.any(cur < n_pts):
            # time range of the last step, :1795-1803
            c_hi, c_lo = dsub(self.t_hi, self.t_lo, self.last_h, np.zeros(n))
            cmp_lt_t = dlt(c_hi, c_lo, self.t_hi, self.t_lo)
            t_lt_cmp = dlt(self.t_hi, self.t_lo, c_hi, c_lo)
            t0h, t0l = np.where(cmp_lt_t, c_hi, self.t_hi), np.where(cmp_lt_t, c_lo, self.t_lo)
            t1h, t1l = np.where(t_lt_cmp, c_hi, self.t_hi), np.where(t_lt_cmp, c_lo, self.t_lo)
            dflags = np.ones(n, dtype=bool)
            while True:  # :1811-1886
                tmp = np.zeros(n)
                for i in range(n):
                    if dflags[i] and cur[i] < n_pts:
                        g = grid[cur[i], i]
                        ge_t0 = not dlt(g, 0.0, t0h[i], t0l[i])
                        le_t1 = not dlt(t1h[i], t1l[i], g, 0.0)
                        dflags[i] = (ge_t0 and le_t1) or (rem_hi[i] == 0 and rem_lo[i] == 0)
                        tmp[i] = g
                    else:
                        dflags[i] = False
                if not dflags.any():
                    break
                tau = dsub(tmp, np.zeros(n), c_hi, c_lo)[0]  # update_d_output(), :2283-2287
                d = self.d_output(tau)
                for i in range(n):
                    if dflags[i]:
                        ret[cur[i], :, i] = d[:, i]
                        cur[i] += 1
                if not np.any(cur < n_pts):
                    break
            if not np.any(cur < n_pts):
                break
            if np.any(self.prop_outcome == STEP_LIMIT):
                break
            # next step, :1899-1913
            lim = np.empty(n)
            for i in range(n):
                if t_dir[i]:
                    lim[i] = rem_hi[i] if dlt(rem_hi[i], rem_lo[i], mdt[i], 0.0) else mdt[i]
                else:
                    lim[i] = rem_hi[i] if dlt(-mdt[i], 0.0, rem_hi[i], rem_lo[i]) else -mdt[i]
            self.step(max_delta_t=lim, write_tc=True)
            nfs = False
            for i in range(n):  # :1922-1971
                oc, h = self.step_outcome[i], self.last_h[i]
                if oc == NF:
                    nfs = True
                else:
                    self.n_steps[i] += int(h != 0)
                    if oc == SUCCESS:
                        self.min_h[i] = min(self.min_h[i], abs(h))
                        self.max_h[i] = max(self.max_h[i], abs(h))
                    if h == rem_hi[i]:
                        rem_hi[i] = rem_lo[i] = 0.0
                    else:
                        r = dsub(grid[-1, i], 0.0, self.t_hi[i], self.t_lo[i])
                        rem_hi[i], rem_lo[i] = r[0][0], r[1][0]
                self.prop_outcome[i] = oc
            if nfs:
                break
            it += 1
            if it == max_steps:
                self.prop_outcome[:] = STEP_LIMIT
        return ret

    def propagate_until_cout(self, t_final, max_delta_t=None, max_steps=0):
        """propagate_until() as the reference's lock-step loop with continuous-output recording
        (src/taylor_adaptive_batch.cpp:1246-1527). Returns an OracleCOut, or None if no iteration completed."""
        import heyoka_b200 as hb
        n = self.n
        tf = np.broadcast_to(np.asarray(t_final, dtype=np.float64), (n,)).copy()
        mdt = np.full(n, np.inf) if max_delta_t is None else np.broadcast_to(np.asarray(max_delta_t, float), (n,))
        SUCCESS, NF, STEP_LIMIT = hb.taylor_outcome.success, hb.taylor_outcome.err_nf_state, hb.taylor_outcome.step_limit

        def dsub(ahi, alo, bhi, blo):
            return hb._dfloat_add(np.atleast_1d(ahi), np.atleast_1d(alo), -np.atleast_1d(bhi), -np.atleast_1d(blo))

        def dlt(ahi, alo, bhi, blo):
            return (ahi < bhi) | ((ahi == bhi) & (alo < blo))

        times_hi, times_lo, tcs = [self.t_hi.copy()], [self.t_lo.copy()], []
        self.n_steps[:] = 0
        self.min_h[:] = np.inf
        self.max_h[:] = 0
        rem_hi, rem_lo = dsub(tf, np.zeros(n), self.t_hi, self.t_lo)
        t_dir = (rem_hi > 0) | ((rem_hi == 0) & (rem_lo >= 0))
        it = 0
        while True:
            lim = np.empty(n)
            for i in range(n):
                if t_dir[i]:
                    lim[i] = rem_hi[i] if dlt(rem_hi[i], rem_lo[i], mdt[i], 0.0) else mdt[i]
                else:
                    lim[i] = rem_hi[i] if dlt(-mdt[i], 0.0, rem_hi[i], rem_lo[i]) else -mdt[i]
            self.step(max_delta_t=lim, write_tc=True)
            n_done, nfs = 0, False
            for i in range(n):
                oc, h = self.step_outcome[i], self.last_h[i]
                if oc == NF:
                    nfs = True
                else:
                    self.n_steps[i] += int(h != 0)
                    if oc == SUCCESS:
                        self.min_h[i] = min(self.min_h[i], abs(h))
                        self.max_h[i] = max(self.max_h[i], abs(h))
                    if h == rem_hi[i]:
                        n_done += 1
                        rem_hi[i] = rem_lo[i] = 0.0
                    else:
                        r = dsub(tf[i], 0.0, self.t_hi[i], self.t_lo[i])
                        rem_hi[i], rem_lo[i] = r[0][0], r[1][0]
                self.prop_outcome[i] = oc
            if nfs:
                break
            times_hi.append(self.t_hi.copy())
            times_lo.append(self.t_lo.copy())
            tcs.append(self.tc.copy())
            it += 1
            if n_done == n:
                break
            if it == max_steps:
                self.prop_outcome[:] = STEP_LIMIT
                break
        if not tcs:
            return None
        times_hi.append(np.where(t_dir, np.inf, -np.inf))
        times_lo.append(np.zeros(n))
        return OracleCOut(self.P, np.array(tcs), np.array(times_hi), np.array(times_lo))


class OracleCOut:
    """Evaluation of a continuous output, src/continuous_output.cpp:640-960 (upper_bound per lane, then Horner /
    compensated summation through the oracle's dense-output function)."""

    def __init__(self, P, tcs, t_hi, t_lo):
        self.P, self.tcs, self.t_hi, self.t_lo = P, tcs, t_hi, t_lo
        self.n = t_hi.shape[1]

    def get_n_steps(self):
        return self.tcs.shape[0]

    def get_bounds(self):
        return self.t_hi[0].copy(), self.t_hi[-2].copy()

    def __call__(self, tm):
        import heyoka_b200 as hb
        tm = np.broadcast_to(np.asarray(tm, dtype=np.float64), (self.n,))
        rows = self.t_hi.shape[0]
        out = np.empty((self.P.n_eq, self.n))

        def lt(ahi, alo, bhi, blo):
            return (ahi < bhi) or (ahi == bhi and alo < blo)

        for i in range(self.n):
            fwd = lt(self.t_hi[0, i], self.t_lo[0, i], self.t_hi[-1, i], self.t_lo[-1, i])
            first, count = 0, rows
            while count:
                step = count // 2
                idx = first + step
                cond = (not lt(tm[i], 0.0, self.t_hi[idx, i], self.t_lo[idx, i])) if fwd else \
                    (not lt(self.t_hi[idx, i], self.t_lo[idx, i], tm[i], 0.0))
                if cond:
                    first, count = idx + 1, count - step - 1
                else:
                    count = step
            k = first - (1 if first != 0 else 0) - (1 if first == rows - 1 else 0)
            h = hb._dfloat_add(np.array([tm[i]]), np.zeros(1), -self.t_hi[k, i:i + 1], -self.t_lo[k, i:i + 1])[0][0]
            tc1 = np.ascontiguousarray(self.tcs[k][:, :, i:i + 1])
            o = np.empty((self.P.n_eq, 1))
            rc = lib.oracle_d_output_w1(_desc_ptr(self.P), C.c_uint32(1), _arr(tc1), _arr(np.array([h])), _arr(o))
            assert rc == 0
            out[:, i] = o[:, 0]
        return out


# ---- event detection (oracle_step_ev_w1) --------------------------------------------------------------------------
class oracle_event(C.Structure):
    _fields_ = [("lane", C.c_uint32), ("idx", C.c_uint32), ("terminal", C.c_int32), ("d_sgn", C.c_int32),
                ("t", C.c_double), ("abs_der", C.c_double)]


class OracleBatch:
    """The surface of heyoka_b200.Batch that an integrator WITH EVENTS uses, served by the CPU oracle. Plugged under
    the product's Python front end (heyoka_b200.taylor_adaptive_batch._make_batch) by OracleEventIntegrator below, so
    that the callback / propagate logic of the front end can be exercised on a machine without a GPU and the device
    kernels can be compared with the oracle step by step."""

    def __init__(self, program, batch, mode=FMA):
        P = self.program = program
        self.n, self.mode = batch, mode
        self.state = np.zeros((P.n_eq, batch))
        self.pars = np.zeros((max(P.n_pars, 1), batch))
        self.t_hi, self.t_lo, self.last_h = np.zeros(batch), np.zeros(batch), np.zeros(batch)
        self._tc = np.zeros((P.n_eq + P.n_ev, P.order + 1, batch))
        self.outcome = np.zeros(batch, dtype=np.int64)
        self._events = []

    def set_kernel(self, **kw):
        pass

    def kernel_info(self):
        return {"tape": "oracle"}

    def check_grid(self, grid, max_delta_t=None):
        pass

    def set_events(self, n_te, dirs, cooldowns, tol):
        self.n_te, self.tol = int(n_te), float(tol)
        self.dirs = np.ascontiguousarray(dirs, dtype=np.int32)
        self.cd_vals = np.ascontiguousarray(list(cooldowns) + [0.0], dtype=np.float64)
        self.cd = np.zeros((self.n, max(self.n_te, 1), 2))
        self.cd_on = np.zeros((self.n, max(self.n_te, 1)), dtype=np.int32)

    def upload(self, state, pars, t_hi, t_lo):
        self.state[...] = state
        if pars is not None:
            self.pars[...] = pars
        self.t_hi[...] = t_hi
        self.t_lo[...] = t_lo

    def download(self):
        return self.state.copy(), self.t_hi.copy(), self.t_lo.copy(), self.last_h.copy()

    def tc(self):
        return self._tc[:self.program.n_eq].copy()

    def tc_events(self, n_ev):
        return self._tc[self.program.n_eq:].copy()

    def step(self, max_delta_t=None, backward=False, write_tc=False):
        n = self.n
        mdt = np.full(n, -np.inf if backward else np.inf) if max_delta_t is None else \
            np.ascontiguousarray(np.broadcast_to(max_delta_t, (n,)), dtype=np.float64)
        cap = 64 * n * max(self.program.n_ev, 1)
        buf = (oracle_event * cap)()
        n_out = C.c_uint32()
        rc = lib.oracle_step_ev_w1(
            _desc_ptr(self.program), C.c_uint32(n), _arr(self.state), _arr(self.pars), _arr(self.t_hi), _arr(self.t_lo),
            _arr(mdt), C.c_double(self.tol), C.c_uint32(self.n_te), self.dirs.ctypes.data_as(C.POINTER(C.c_int32)),
            _arr(self.cd_vals), _arr(self.cd), self.cd_on.ctypes.data_as(C.POINTER(C.c_int32)), _arr(self._tc),
            _arr(self.last_h), self.outcome.ctypes.data_as(C.POINTER(C.c_int64)), buf, C.c_uint32(cap), C.byref(n_out),
            C.c_int(self.mode))
        assert rc == 0, rc
        self._events = [(e.lane, e.idx, bool(e.terminal), e.d_sgn, e.t, e.abs_der) for e in buf[:n_out.value]]

    def step_res(self):
        return self.outcome.copy(), self.last_h.copy()

    def events(self):
        return list(self._events)

    def reset_cooldowns(self, lane=-1):
        if lane >= self.n:  # (hy_batch_reset_cooldowns(), src/taylor_adaptive_batch.cpp:2348-2352)
            raise ValueError("Cannot reset the cooldowns at batch index %d: the batch size for this integrator is only %d"
                             % (lane, self.n))
        if lane < 0:
            self.cd_on[...] = 0
        else:
            self.cd_on[lane] = 0

    def cooldowns(self, n_te):
        return (self.cd_on.T[:n_te].astype(np.uint8), self.cd[:, :, 0].T[:n_te].copy(), self.cd[:, :, 1].T[:n_te].copy())

    def d_output(self, tau):
        P = self.program
        tau = np.ascontiguousarray(np.broadcast_to(tau, (self.n,)), dtype=np.float64)
        out = np.empty((P.n_eq, self.n))
        tc = np.ascontiguousarray(self._tc[:P.n_eq])
        rc = lib.oracle_d_output_w1(_desc_ptr(P), C.c_uint32(self.n), _arr(tc), _arr(tau), _arr(out))
        assert rc == 0
        return out


def ev_max_depth(reset=True):
    """Deepest working list of the oracle's root isolation (entries held at once) since the last reset; the device
    holds that list in a stack of dev::EV_STACK entries."""
    lib.oracle_ev_max_depth_w1.restype = C.c_uint32
    return int(lib.oracle_ev_max_depth_w1(C.c_int(1 if reset else 0)))


_OEI = None


def OracleEventIntegrator(*args, mode=FMA, **kw):
    """heyoka_b200.taylor_adaptive_batch (the product's host-side front end: callbacks, lock-step propagation) over the
    CPU oracle instead of the device."""
    global _OEI
    if _OEI is None:
        import heyoka_b200 as hb

        class _Impl(hb.taylor_adaptive_batch):
            def __init__(self, *a, mode=FMA, **k):
                self._oracle_mode = mode
                super().__init__(*a, **k)

            def _make_batch(self, P, batch_size, device):
                return OracleBatch(P, batch_size, self._oracle_mode)

        _OEI = _Impl
    return _OEI(*args, mode=mode, **kw)
