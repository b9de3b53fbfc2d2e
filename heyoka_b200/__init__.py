"""heyoka_b200 — H100-native batch Taylor integrator (drop-in for heyoka's taylor_adaptive_batch<double>).

This Python package is a thin ctypes mirror of the C ABI in include/heyoka_b200.h, shaped after the
reference's C++ API (include/heyoka/taylor.hpp:780-1121) so that the parity tests read like the
reference's own tests (test/taylor_adaptive_batch.cpp). The product is the native library
(heyoka_b200/lib/libheyoka_b200.so: host C++ front end + hand-written sm_90a CUDA kernels); there is no
Python or CPU fallback for the compute path: if the library is missing, importing fails loudly.
"""
import ctypes as C
import enum
import os

import numpy as np

from . import _capi
from ._capi import lib, check, HyError  # noqa: F401

__all__ = [
    "expression", "make_vars", "par", "time", "sin", "cos", "tanh", "exp", "log", "sigmoid", "relu", "relup", "sqrt", "square", "pow", "sum",
    "prod", "diff", "var_args", "var_ode_sys", "model", "taylor_adaptive_batch", "t_event_batch", "nt_event_batch", "event_direction", "continuous_output_batch", "taylor_outcome", "Program", "Batch", "order_from_tol", "HyError",
]


class taylor_outcome:
    """include/heyoka/taylor.hpp:142-155."""
    success = -4294967297
    step_limit = -4294967298
    time_limit = -4294967299
    err_nf_state = -4294967300
    cb_stop = -4294967301


# ------------------------------------------------------------------------------------------------
# Expressions
# ------------------------------------------------------------------------------------------------
class expression:
    __slots__ = ("_h",)

    def __init__(self, value=0.0, _handle=None):
        if _handle is not None:
            self._h = int(_handle.value if isinstance(_handle, C.c_void_p) else _handle)
        elif isinstance(value, expression):
            self._h = _capi.ex_checked(lib.hy_ex_copy(value._h))
        elif isinstance(value, str):
            self._h = _capi.ex_checked(lib.hy_ex_var(value.encode()))
        else:
            self._h = _capi.ex_checked(lib.hy_ex_num(float(value)))

    def __del__(self):
        h = getattr(self, "_h", None)
        if h and lib is not None:
            lib.hy_ex_free(h)
            self._h = None

    @staticmethod
    def _wrap(x):
        return x if isinstance(x, expression) else expression(x)

    def _bin(self, op, other, swap=False):
        o = expression._wrap(other)
        a, b = (o, self) if swap else (self, o)
        return expression(_handle=_capi.ex_checked(lib.hy_ex_binary(op.encode(), a._h, b._h)))

    def __add__(self, o):
        return self._bin("+", o)

    def __radd__(self, o):
        return self._bin("+", o, True)

    def __sub__(self, o):
        return self._bin("-", o)

    def __rsub__(self, o):
        return self._bin("-", o, True)

    def __mul__(self, o):
        return self._bin("*", o)

    def __rmul__(self, o):
        return self._bin("*", o, True)

    def __truediv__(self, o):
        return self._bin("/", o)

    def __rtruediv__(self, o):
        return self._bin("/", o, True)

    def __pow__(self, o):
        return self._bin("^", o)

    def __neg__(self):
        return expression(_handle=_capi.ex_checked(lib.hy_ex_binary(b"n", self._h, None)))

    def __pos__(self):
        return self

    def __repr__(self):
        n = lib.hy_ex_str(self._h, None, 0)
        buf = C.create_string_buffer(n + 1)
        lib.hy_ex_str(self._h, buf, n + 1)
        return buf.value.decode()


def _func(name, *args):
    keep = [expression._wrap(a) for a in args]  # keep temporaries alive
    arr = (C.c_void_p * len(keep))(*[k._h for k in keep])
    return expression(_handle=_capi.ex_checked(lib.hy_ex_func(name.encode(), arr, len(keep))))


def make_vars(*names):
    return tuple(expression(n) for n in names)


class _Par:
    def __getitem__(self, idx):
        return expression(_handle=_capi.ex_checked(lib.hy_ex_par(int(idx))))


par = _Par()
time = expression(_handle=_capi.ex_checked(lib.hy_ex_time()))


def sin(e):
    return _func("sin", e)


def cos(e):
    return _func("cos", e)


def tanh(e):
    return _func("tanh", e)


def exp(e):
    return _func("exp", e)


def sigmoid(e):
    return _func("sigmoid", e)


def relu(e, slope=0.0):
    """relu(x) / leaky ReLU (src/math/relu.cpp); slope must be finite and non-negative."""
    return _func("relu", e) if slope == 0 else _func("leaky_relu", e, float(slope))


def relup(e, slope=0.0):
    """Derivative of the (leaky) ReLU: 1 for x > 0, slope otherwise (src/math/relu.cpp)."""
    return _func("relup", e, float(slope))


def log(e):
    return _func("log", e)


def sqrt(e):
    return _func("sqrt", e)


def square(e):
    return _func("square", e)


def pow(b, e):  # noqa: A001
    return expression._wrap(b) ** e


def sum(terms):  # noqa: A001
    return _func("sum", *terms)


def prod(terms):
    return _func("prod", *terms)


def diff(e, wrt):
    """Symbolic derivative of e with respect to a variable or a parameter par[i] (folded like every builder)."""
    e, wrt = expression._wrap(e), expression._wrap(wrt)
    return expression(_handle=_capi.ex_checked(lib.hy_ex_diff(e._h, wrt._h)))


class var_args(enum.IntFlag):
    """Arguments of the variational equations: the state variables (LHS order), the parameters (index order), the
    initial time (not implemented). vars | params: the state variables first."""
    vars = 1
    params = 2
    time = 4
    all = 7


class var_ode_sys:
    """An ODE system augmented with its first-order variational equations (heyoka_b200/var_ode_sys.hpp).

    args: var_args flags, or a list of state variables and / or parameters, kept in the order given. The augmented
    state is [x_0 .. x_{n-1}, dx_0/da_0 .. dx_0/da_{m-1}, dx_1/da_0, ...]: state[n:] reshaped to (n, m) is the STM."""

    def __init__(self, sys, args=var_args.vars, order=1):
        keep = [(expression._wrap(lhs), expression._wrap(rhs)) for lhs, rhs in sys]
        n = len(keep)
        lhs = (C.c_void_p * max(n, 1))(*[p[0]._h for p in keep])
        rhs = (C.c_void_p * max(n, 1))(*[p[1]._h for p in keep])
        if isinstance(args, int):
            flags, items = int(args), []  # (no flags: an empty explicit list, refused by the native code)
        else:
            flags, items = 0, [expression._wrap(a) for a in args]
        arr = (C.c_void_p * max(len(items), 1))(*[a._h for a in items])
        n_eq, n_args = C.c_uint32(), C.c_uint32()
        call = lambda ol, orr, oa: lib.hy_var_ode_sys(lhs, rhs, n, flags, arr, len(items), int(order),  # noqa: E731
                                                      C.byref(n_eq), C.byref(n_args), ol, orr, oa)
        check(call(None, None, None))
        ol, orr, oa = (C.c_void_p * n_eq.value)(), (C.c_void_p * n_eq.value)(), (C.c_void_p * n_args.value)()
        check(call(ol, orr, oa))
        self.sys = [(expression(_handle=ol[i]), expression(_handle=orr[i])) for i in range(n_eq.value)]
        self.vargs = [expression(_handle=oa[j]) for j in range(n_args.value)]
        self.n_orig_sv = n
        self.order = int(order)


class model:
    """model::nbody / pendulum / ffnn (src/model/*.cpp)."""

    @staticmethod
    def nbody(n, masses=None, Gconst=1.0):
        lhs = (C.c_void_p * (6 * n))()
        rhs = (C.c_void_p * (6 * n))()
        if masses is None:
            check(lib.hy_model_nbody(n, None, 0, float(Gconst), lhs, rhs))
        else:
            m = np.ascontiguousarray(masses, dtype=np.float64)
            check(lib.hy_model_nbody(n, m.ctypes.data_as(C.POINTER(C.c_double)), len(m), float(Gconst), lhs, rhs))
        return [(expression(_handle=lhs[i]), expression(_handle=rhs[i])) for i in range(6 * n)]

    @staticmethod
    def pendulum(gconst=1.0, length=1.0):
        lhs = (C.c_void_p * 2)()
        rhs = (C.c_void_p * 2)()
        check(lib.hy_model_pendulum(float(gconst), float(length), lhs, rhs))
        return [(expression(_handle=lhs[i]), expression(_handle=rhs[i])) for i in range(2)]

    @staticmethod
    def ffnn(inputs, nn_hidden, n_out, activations, nn_wb=None):
        ids = {"identity": 0, "tanh": 1, "sin": 2, "exp": 3, "sigmoid": 4, "relu": 5}
        ins = [expression._wrap(i) for i in inputs]
        arr = (C.c_void_p * len(ins))(*[i._h for i in ins])
        hid = (C.c_uint32 * len(nn_hidden))(*nn_hidden)
        act = (C.c_int * len(activations))(*[ids[a] for a in activations])
        out = (C.c_void_p * n_out)()
        if nn_wb is None:
            check(lib.hy_model_ffnn(arr, len(ins), hid, len(nn_hidden), n_out, act, None, 0, out))
        else:
            wb = np.ascontiguousarray(nn_wb, dtype=np.float64)
            check(lib.hy_model_ffnn(arr, len(ins), hid, len(nn_hidden), n_out, act,
                                    wb.ctypes.data_as(C.POINTER(C.c_double)), len(wb), out))
        return [expression(_handle=out[i]) for i in range(n_out)]


def order_from_tol(tol):
    o = C.c_uint32()
    check(lib.hy_order_from_tol(float(tol), C.byref(o)))
    return o.value


# ------------------------------------------------------------------------------------------------
# Program
# ------------------------------------------------------------------------------------------------
class Program:
    """The lowered Taylor decomposition of an ODE system (include/heyoka_b200.h, section B)."""

    def __init__(self, sys, tol=0.0, high_accuracy=False, _handle=None, events=()):
        """events: the event equations (terminal events first), decomposed together with the system like
        taylor_add_adaptive_step_with_events() does (src/taylor_00.cpp:605)."""
        if _handle is not None:
            self._h = _handle
        else:
            if isinstance(sys, var_ode_sys):
                sys = sys.sys  # (the augmented system is an ordinary ODE system for the stepper)
            n = len(sys)
            self._keep = [(expression._wrap(lhs), expression._wrap(rhs)) for lhs, rhs in sys]
            self._keep_ev = [expression._wrap(e) for e in events]
            lhs = (C.c_void_p * n)(*[p[0]._h for p in self._keep])
            rhs = (C.c_void_p * n)(*[p[1]._h for p in self._keep])
            evs = (C.c_void_p * max(len(self._keep_ev), 1))(*[e._h for e in self._keep_ev])
            h = C.c_void_p()
            check(lib.hy_program_from_sys_ev(lhs, rhs, n, evs, len(self._keep_ev), float(tol), int(bool(high_accuracy)),
                                             C.byref(h)))
            self._h = h
        d = _capi.hy_program_desc()
        check(lib.hy_program_get_desc(self._h, C.byref(d)))
        self.desc = d
        self.n_eq, self.n_uvars, self.n_pars, self.order = d.n_eq, d.n_uvars, d.n_pars, d.order
        self.high_accuracy = bool(d.high_accuracy)
        self.n_ev = d.n_ev

    def ev_defs(self):
        return np.ctypeslib.as_array(C.cast(self.desc.ev_defs, C.POINTER(C.c_uint32)), shape=(self.n_ev,)).copy() \
            if self.n_ev else np.zeros(0, dtype=np.uint32)

    @classmethod
    def from_arrays(cls, n_eq, n_uvars, n_pars, order, ops, args, consts, sv_defs, high_accuracy=False):
        ops = np.ascontiguousarray(ops, dtype=np.uint32).reshape(-1, 4)
        args = np.ascontiguousarray(args, dtype=np.uint32)
        consts = np.ascontiguousarray(consts, dtype=np.float64)
        sv_defs = np.ascontiguousarray(sv_defs, dtype=np.uint32)
        d = _capi.hy_program_desc()
        d.n_eq, d.n_uvars, d.n_pars, d.order = n_eq, n_uvars, n_pars, order
        d.n_args, d.n_consts, d.high_accuracy = len(args), len(consts), int(high_accuracy)
        d.ops = ops.ctypes.data_as(C.c_void_p)
        d.args = args.ctypes.data_as(C.c_void_p)
        d.consts = consts.ctypes.data_as(C.c_void_p)
        d.sv_defs = sv_defs.ctypes.data_as(C.c_void_p)
        h = C.c_void_p()
        check(lib.hy_program_create(C.byref(d), C.byref(h)))
        return cls(None, _handle=h)

    def __del__(self):
        h = getattr(self, "_h", None)
        if h and lib is not None:
            lib.hy_program_destroy(h)
            self._h = None

    @property
    def dc_size(self):
        return lib.hy_program_dc_size(self._h)

    def dc_str(self):
        n = lib.hy_program_dc_str(self._h, None, 0)
        buf = C.create_string_buffer(n + 1)
        lib.hy_program_dc_str(self._h, buf, n + 1)
        return buf.value.decode()

    def costs(self):
        a, b, c = C.c_double(), C.c_double(), C.c_double()
        check(lib.hy_program_costs(self._h, C.byref(a), C.byref(b), C.byref(c)))
        return {"b_min": a.value, "b_tape": b.value, "flops": c.value}

    def ops_array(self):
        n = self.n_uvars - self.n_eq
        return np.ctypeslib.as_array(C.cast(self.desc.ops, C.POINTER(C.c_uint32)), shape=(n, 4)).copy()


# ------------------------------------------------------------------------------------------------
# Batch (device-resident)
# ------------------------------------------------------------------------------------------------
def _dptr(a):
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_double))


class Batch:
    """Device-resident integrator state + kernels (include/heyoka_b200.h, section C)."""

    def __init__(self, program, batch, device=-1):
        """device: a CUDA ordinal (-1 = current device), or a list of ordinals / "all" to shard the lanes over several
        GPUs of the box (hy_batch_create_multi(): contiguous blocks of lanes, one host thread per device)."""
        self.program = program
        self.n = int(batch)
        h = C.c_void_p()
        if isinstance(device, str) or hasattr(device, "__len__"):
            devs = [] if isinstance(device, str) else [int(d) for d in device]
            arr = (C.c_int * len(devs))(*devs) if devs else None
            check(lib.hy_batch_create_multi(program._h, self.n, arr, len(devs), C.byref(h)))
        else:
            check(lib.hy_batch_create(program._h, self.n, int(device), C.byref(h)))
        self._h = h

    @property
    def n_shards(self):
        return lib.hy_batch_n_shards(self._h)

    def __del__(self):
        h = getattr(self, "_h", None)
        if h and lib is not None:
            lib.hy_batch_destroy(h)
            self._h = None

    def set_stream(self, cuda_stream):
        check(lib.hy_batch_set_stream(self._h, C.c_void_p(int(cuda_stream))))

    def set_launch_config(self, block_threads=0, blocks_per_sm=0):
        check(lib.hy_batch_set_launch_config(self._h, int(block_threads), int(blocks_per_sm)))

    def set_kernel(self, tape="auto", lanes_per_warp=0, lanes_per_thread=0, block_threads=0, blocks_per_sm=0):
        # "nbody" / "nbody-cta": the dedicated N-body kernel (warp / CTA teams; lanes_per_thread is ignored).
        # "smem-notmem" is the same as "smem" (kept for compatibility).
        # "nn": the dense-network kernel (right-hand sides that are feed-forward networks).
        mode = {"auto": 0, "hbm": 1, "smem": 2, "smem-notmem": 3, "global": 4, "global-cta": 5, "nbody": 6,
                "nbody-cta": 7, "nn": 8, "nbody-lane": 9}[tape]
        check(lib.hy_batch_set_kernel(self._h, mode, int(lanes_per_warp), int(lanes_per_thread), int(block_threads),
                                      int(blocks_per_sm)))

    def kernel_info(self):
        ki = _capi.hy_kernel_info()
        check(lib.hy_batch_get_kernel(self._h, C.byref(ki)))
        d = {f[0]: getattr(ki, f[0]) for f in ki._fields_}
        d["tape"] = {1: "hbm", 2: "smem", 4: "global", 5: "global-cta", 6: "nbody", 7: "nbody-cta", 8: "nn", 9: "nbody-lane"}.get(ki.tape_mode, "?")
        return d

    def sync(self):
        check(lib.hy_batch_sync(self._h))

    def upload(self, state=None, pars=None, t_hi=None, t_lo=None):
        f = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float64)  # noqa: E731
        s, p, th, tl = f(state), f(pars), f(t_hi), f(t_lo)
        check(lib.hy_batch_upload(self._h, _dptr(s), _dptr(p), _dptr(th), _dptr(tl)))

    def download(self):
        P = self.program
        state = np.empty((P.n_eq, self.n))
        t_hi, t_lo, last_h = np.empty(self.n), np.empty(self.n), np.empty(self.n)
        check(lib.hy_batch_download(self._h, _dptr(state), _dptr(t_hi), _dptr(t_lo), _dptr(last_h)))
        return state, t_hi, t_lo, last_h

    def step_res(self):
        oc, h = np.empty(self.n, dtype=np.int64), np.empty(self.n)
        check(lib.hy_batch_download_step_res(self._h, oc.ctypes.data_as(C.POINTER(C.c_int64)), _dptr(h)))
        return oc, h

    def prop_res(self):
        oc = np.empty(self.n, dtype=np.int64)
        mn, mx = np.empty(self.n), np.empty(self.n)
        ns = np.empty(self.n, dtype=np.uint64)
        check(lib.hy_batch_download_prop_res(self._h, oc.ctypes.data_as(C.POINTER(C.c_int64)), _dptr(mn), _dptr(mx),
                                             ns.ctypes.data_as(C.POINTER(C.c_uint64))))
        return oc, mn, mx, ns

    def tc(self):
        P = self.program
        out = np.empty((P.n_eq, P.order + 1, self.n))
        check(lib.hy_batch_download_tc(self._h, _dptr(out)))
        return out

    def ptrs(self):
        p = _capi.hy_batch_ptrs()
        check(lib.hy_batch_get_ptrs(self._h, C.byref(p)))
        return p

    def step(self, max_delta_t=None, backward=False, write_tc=False):
        m = None if max_delta_t is None else np.ascontiguousarray(max_delta_t, dtype=np.float64)
        check(lib.hy_batch_step(self._h, _dptr(m), 0, int(backward), int(write_tc)))

    def propagate_until(self, t_hi, t_lo=None, max_delta_t=None, max_steps=0, write_tc=False):
        f = lambda a: None if a is None else np.ascontiguousarray(np.broadcast_to(a, (self.n,)), dtype=np.float64)  # noqa
        th, tl, m = f(t_hi), f(t_lo), f(max_delta_t)
        check(lib.hy_batch_propagate_until(self._h, _dptr(th), _dptr(tl), _dptr(m), int(max_steps), int(write_tc)))

    def propagate_until_host(self, state, t_hi, t_lo, t_final, t_final_lo=None, max_delta_t=None, max_steps=0, pars=None):
        """hy_batch_propagate_until_host(): upload, propagate, download in one call. state [n_eq, batch], t_hi, t_lo
        [batch] (C-contiguous float64) are overwritten in place; returns (last_h, outcome, min_h, max_h, n_steps)."""
        for a in (state, t_hi, t_lo):
            assert a.dtype == np.float64 and a.flags["C_CONTIGUOUS"]
        assert state.shape == (self.program.n_eq, self.n) and t_hi.shape == (self.n,) and t_lo.shape == (self.n,)
        f = lambda a: None if a is None else np.ascontiguousarray(np.broadcast_to(a, (self.n,)), dtype=np.float64)  # noqa
        tf, tfl, m = f(t_final), f(t_final_lo), f(max_delta_t)
        pr = None if pars is None else np.ascontiguousarray(pars, dtype=np.float64)
        last_h, mn, mx = np.empty(self.n), np.empty(self.n), np.empty(self.n)
        oc, ns = np.empty(self.n, dtype=np.int64), np.empty(self.n, dtype=np.uint64)
        check(lib.hy_batch_propagate_until_host(self._h, _dptr(state), _dptr(pr), _dptr(t_hi), _dptr(t_lo), _dptr(tf),
                                                _dptr(tfl), _dptr(m), int(max_steps), _dptr(state), _dptr(t_hi),
                                                _dptr(t_lo), _dptr(last_h),
                                                oc.ctypes.data_as(C.POINTER(C.c_int64)), _dptr(mn), _dptr(mx),
                                                ns.ctypes.data_as(C.POINTER(C.c_uint64))))
        return last_h, oc, mn, mx, ns

    def propagate_until_dev(self, d_t_hi, d_t_lo=0, d_max_delta_t=0, max_steps=0, write_tc=False):
        flag = C.c_int()
        vp = lambda x: C.cast(C.c_void_p(int(x) if x else None), C.POINTER(C.c_double))  # noqa: E731
        check(lib.hy_batch_propagate_until_dev(self._h, vp(d_t_hi), vp(d_t_lo), vp(d_max_delta_t), int(max_steps),
                                               int(write_tc), C.byref(flag)))
        return flag.value

    def propagate_until_cout(self, t_hi, t_lo=None, max_delta_t=None, max_steps=0, step_cb=None):
        """propagate_until() with continuous output (lock-step loop); returns a continuous_output_batch or None.
        step_cb: callable() -> int run after every recorded iteration (> 0 continue, 0 stop with cb_stop, < 0 abort:
        hy_batch_propagate_until_cout_cb)."""
        f = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float64)  # noqa: E731
        th, tl, md = f(t_hi), f(t_lo), f(max_delta_t)
        h = C.c_void_p()
        if step_cb is None:
            check(lib.hy_batch_propagate_until_cout(self._h, _dptr(th), None if tl is None else _dptr(tl),
                                                    None if md is None else _dptr(md), int(max_steps), C.byref(h)))
        else:
            tramp = C.CFUNCTYPE(C.c_int, C.c_void_p)(lambda _user: int(step_cb()))
            st = lib.hy_batch_propagate_until_cout_cb(self._h, _dptr(th), None if tl is None else _dptr(tl),
                                                      None if md is None else _dptr(md), int(max_steps),
                                                      C.cast(tramp, C.c_void_p), None, C.byref(h))
            if st == _capi.HY_ERR_CALLBACK:
                return None  # (the caller re-raises what its callback raised)
            check(st)
        return continuous_output_batch(h, self.program.n_eq, self.n, self.program.order) if h.value else None

    def propagate_grid(self, grid, max_delta_t=None, max_steps=0):
        """grid: [n_pts, batch]; returns the states at the grid points, [n_pts, n_eq, batch] (NaN where not reached)."""
        grid = np.ascontiguousarray(grid, dtype=np.float64)
        n_pts = grid.size // self.n
        md = None if max_delta_t is None else np.ascontiguousarray(max_delta_t, dtype=np.float64)
        out = np.empty((n_pts, self.program.n_eq, self.n))
        check(lib.hy_batch_propagate_grid(self._h, _dptr(grid), n_pts, None if md is None else _dptr(md),
                                          int(max_steps), _dptr(out)))
        return out

    def d_output(self, tau):
        P = self.program
        tau = np.ascontiguousarray(np.broadcast_to(tau, (self.n,)), dtype=np.float64)
        out = np.empty((P.n_eq, self.n))
        check(lib.hy_batch_d_output(self._h, _dptr(tau), _dptr(out)))
        return out

    def eval_taylor_map(self, n_orig_sv, dx, out=None):
        """Taylor map x + Phi dx of the resident state (hy_batch_eval_taylor_map()): dx [n_args, batch] on the host,
        returns out [n_orig_sv, batch]."""
        dx = np.ascontiguousarray(dx, dtype=np.float64).reshape(-1, self.n)
        out = np.empty((n_orig_sv, self.n)) if out is None else out
        assert out.dtype == np.float64 and out.flags["C_CONTIGUOUS"] and out.size == n_orig_sv * self.n
        check(lib.hy_batch_eval_taylor_map(self._h, int(n_orig_sv), dx.shape[0], _dptr(dx), _dptr(out), 0))
        return out

    def eval_taylor_map_dev(self, n_orig_sv, n_args, d_dx, d_out):
        """The same on device pointers (ints, e.g. torch data_ptr()), enqueued on the batch's stream."""
        vp = lambda x: C.cast(C.c_void_p(int(x)), C.POINTER(C.c_double))  # noqa: E731
        check(lib.hy_batch_eval_taylor_map(self._h, int(n_orig_sv), int(n_args), vp(d_dx), vp(d_out), 1))

    # --- events (include/heyoka_b200.h, section E) ---
    def set_events(self, n_te, dirs, cooldowns, tol):
        d = np.ascontiguousarray(dirs, dtype=np.int32)
        c = np.ascontiguousarray(cooldowns, dtype=np.float64)
        check(lib.hy_batch_set_events(self._h, int(n_te), d.ctypes.data_as(C.POINTER(C.c_int32)), _dptr(c), float(tol)))

    def events(self):
        """Events of the last step as (lane, idx, terminal, d_sgn, t, abs_der) tuples, in callback order."""
        n = lib.hy_batch_n_events(self._h)
        buf = (_capi.hy_event_rec * max(n, 1))()
        check(lib.hy_batch_get_events(self._h, buf, n))
        return [(r.lane, r.idx, bool(r.terminal), r.d_sgn, r.t, r.abs_der) for r in buf[:n]]

    def reset_cooldowns(self, lane=-1):
        check(lib.hy_batch_reset_cooldowns(self._h, int(lane)))

    def cooldowns(self, n_te):
        a = np.zeros((max(n_te, 1), self.n), dtype=np.uint8)
        s, c = np.zeros((max(n_te, 1), self.n)), np.zeros((max(n_te, 1), self.n))
        check(lib.hy_batch_get_cooldowns(self._h, a.ctypes.data_as(C.POINTER(C.c_uint8)), _dptr(s), _dptr(c)))
        return a[:n_te], s[:n_te], c[:n_te]

    def tc_events(self, n_ev):
        """Taylor coefficients of the event equations of the last step, [n_ev, order + 1, batch] (device rows n_eq..)."""
        out = np.empty((n_ev, self.program.order + 1, self.n))
        check(lib.hy_batch_download_tc_events(self._h, _dptr(out)))
        return out

    def check_grid(self, grid, max_delta_t=None):
        g = np.ascontiguousarray(grid, dtype=np.float64)
        m = None if max_delta_t is None else np.ascontiguousarray(max_delta_t, dtype=np.float64)
        check(lib.hy_batch_check_grid(self._h, _dptr(g), g.shape[0], _dptr(m)))

    def launch_count(self):
        n = C.c_uint64()
        check(lib.hy_batch_launch_count(self._h, C.byref(n)))
        return n.value


# ------------------------------------------------------------------------------------------------
# taylor_adaptive_batch: host-mirrored integrator with the reference's surface.
# ------------------------------------------------------------------------------------------------
class continuous_output_batch:
    """Continuous output of a propagate_until() (include/heyoka/continuous_output.hpp): callable with one time or
    one time per lane, returns the state [n_eq, batch] at those times (dense output of the step that contains them)."""

    def __init__(self, handle, n_eq, batch, order):
        self._h, self._n_eq, self._n, self._order = handle, n_eq, batch, order
        self._output = np.zeros((n_eq, batch))

    def __del__(self):
        if getattr(self, "_h", None):
            lib.hy_cout_destroy(self._h)
            self._h = None

    def __call__(self, tm):
        t = np.ascontiguousarray(np.broadcast_to(np.asarray(tm, dtype=np.float64), (self._n,)))
        check(lib.hy_cout_eval(self._h, _dptr(t), _dptr(self._output)))
        return self._output

    @property
    def output(self):
        return self._output

    def get_bounds(self):
        lb, ub = np.empty(self._n), np.empty(self._n)
        check(lib.hy_cout_get_bounds(self._h, _dptr(lb), _dptr(ub)))
        return lb, ub

    def get_n_steps(self):
        return int(lib.hy_cout_n_steps(self._h))

    def get_batch_size(self):
        return self._n

    def get_times(self):
        """The times at the ends of the recorded iterations, [n_steps + 2, batch]: row 0 = the starting times, last row =
        the +-infinity padding (get_times(), src/continuous_output.cpp:1157-1163)."""
        out = np.empty((self.get_n_steps() + 2, self._n))
        check(lib.hy_cout_download(self._h, _dptr(out), None, None))
        return out

    def get_tcs(self):
        """The Taylor coefficients of the recorded iterations, [n_steps, n_eq, order + 1, batch] (get_tcs(), :1165-1169)."""
        out = np.empty((self.get_n_steps(), self._n_eq, self._order + 1, self._n))
        check(lib.hy_cout_download(self._h, None, None, _dptr(out)))
        return out


class event_direction:
    """include/heyoka/events.hpp:40-47."""
    negative = -1
    any = 0
    positive = 1


class t_event_batch:
    """Terminal event of a batch integrator (include/heyoka/events.hpp:52-118): callback(ta, d_sgn, batch_idx) -> bool
    (True: the integration may continue), cooldown < 0 = automatic."""

    def __init__(self, ex, callback=None, cooldown=-1.0, direction=event_direction.any):
        self.ex = expression._wrap(ex)
        self.callback = callback
        cooldown = float(cooldown)
        if not np.isfinite(cooldown):
            raise ValueError("Cannot set a non-finite cooldown value for a terminal event")
        if direction not in (-1, 0, 1):
            raise ValueError("Invalid value selected for the direction of a terminal event")
        self.cooldown, self.direction = cooldown, int(direction)


class nt_event_batch:
    """Non-terminal event of a batch integrator (include/heyoka/events.hpp:142-196): callback(ta, t, d_sgn, batch_idx)."""

    def __init__(self, ex, callback, direction=event_direction.any):
        self.ex = expression._wrap(ex)
        if callback is None:
            raise ValueError("Cannot construct a non-terminal event with an empty callback")
        if direction not in (-1, 0, 1):
            raise ValueError("Invalid value selected for the direction of a non-terminal event")
        self.callback, self.direction = callback, int(direction)


class taylor_adaptive_batch:
    """Mirror of heyoka::taylor_adaptive_batch<double> (include/heyoka/taylor.hpp:780-1121).

    The integrator owns host arrays (state [n_eq, batch], pars [n_pars, batch], time) that the user may
    modify between calls; like the reference's raw-pointer contract they are re-uploaded at every
    step()/propagate_*() entry and refreshed on exit.
    """

    def __init__(self, sys, state, batch_size, time=0.0, tol=0.0, high_accuracy=False, compact_mode=False, pars=None,
                 device=-1, t_events=None, nt_events=None, parallel_mode=False, kernel=None):
        batch_size = int(batch_size)
        if batch_size == 0:
            raise ValueError("The batch size in an adaptive Taylor integrator cannot be zero")
        self._tes, self._ntes = list(t_events or []), list(nt_events or [])
        self._with_events = bool(self._tes or self._ntes)
        self._vsys = sys if isinstance(sys, var_ode_sys) else None
        self._prog = Program(sys, tol=tol, high_accuracy=high_accuracy,
                             events=[e.ex for e in self._tes] + [e.ex for e in self._ntes])
        P = self._prog
        state = np.array(state, dtype=np.float64)
        if self._vsys is not None and state.size in (0, self._vsys.n_orig_sv * batch_size):
            state = _var_initial_state(self._vsys, state, batch_size)
        self._tstate = None if self._vsys is None else np.zeros((self._vsys.n_orig_sv, batch_size))
        # Size checks of finalise_ctor_impl(), src/taylor_adaptive_batch.cpp:164-274.
        if state.size != P.n_eq * batch_size:
            raise ValueError(
                "Inconsistent sizes detected in the initialization of an adaptive Taylor integrator in batch mode: "
                "the state vector has a dimension of %d and a batch size of %d, while the number of equations is %d"
                % (state.size, batch_size, P.n_eq))
        self._state = state.reshape(P.n_eq, batch_size).copy()
        tm = np.broadcast_to(np.asarray(time, dtype=np.float64), (batch_size,)) if np.ndim(time) == 0 else \
            np.asarray(time, dtype=np.float64)
        if tm.size != batch_size:
            raise ValueError(
                "Invalid initial time vector specified in the construction of an adaptive Taylor integrator in batch "
                "mode: the batch size is %d, but the number of specified initial times is %d" % (batch_size, tm.size))
        if not np.all(np.isfinite(self._state)):
            raise ValueError("A non-finite value was detected in the initial state of an adaptive Taylor integrator")
        if not np.all(np.isfinite(tm)):
            raise ValueError("A non-finite initial time was detected in the initialisation of an adaptive Taylor "
                             "integrator")
        self._t_hi = tm.copy()
        self._t_lo = np.zeros(batch_size)
        if pars is None:
            self._pars = np.zeros((P.n_pars, batch_size))
        else:
            pars = np.array(pars, dtype=np.float64)
            if pars.size != P.n_pars * batch_size:
                raise ValueError(
                    "Invalid number of parameter values passed to the constructor of an adaptive Taylor integrator in "
                    "batch mode: %d parameter value(s) were passed, but the ODE system contains %d parameter(s) (in "
                    "batches of %d)" % (pars.size, P.n_pars, batch_size))
            self._pars = pars.reshape(P.n_pars, batch_size).copy()
        self._tol = float(tol) if tol > 0 else float(np.finfo(np.float64).eps)
        self._batch_size = batch_size
        self._compact_mode = bool(compact_mode)
        self._b = self._make_batch(P, batch_size, device)
        if kernel is not None:
            self._b.set_kernel(**kernel)
        if self._with_events:
            self._b.set_events(len(self._tes), [e.direction for e in self._tes] + [e.direction for e in self._ntes],
                               [e.cooldown for e in self._tes], self._tol)
        self._last_h = np.zeros(batch_size)
        self._step_res = None
        self._prop_res = None
        self._tc = None

    def _make_batch(self, P, batch_size, device):
        return Batch(P, batch_size, device)

    # --- getters -------------------------------------------------------------------------------
    def get_batch_size(self):
        return self._batch_size

    def get_order(self):
        return self._prog.order

    def get_tol(self):
        return self._tol

    def get_high_accuracy(self):
        return self._prog.high_accuracy

    def get_compact_mode(self):
        return self._compact_mode

    def get_dim(self):
        return self._prog.n_eq

    @property
    def state(self):
        return self._state

    @property
    def pars(self):
        return self._pars

    @property
    def time(self):
        return self._t_hi

    @property
    def dtime(self):
        return self._t_hi, self._t_lo

    def set_time(self, t):
        t = np.broadcast_to(np.asarray(t, dtype=np.float64), (self._batch_size,)) if np.ndim(t) == 0 else np.asarray(t)
        if t.size != self._batch_size:
            raise ValueError("Invalid number of new times specified in a Taylor integrator in batch mode: the batch "
                             "size is %d, but the number of specified times is %d" % (self._batch_size, t.size))
        self._t_hi = np.array(t, dtype=np.float64)
        self._t_lo = np.zeros(self._batch_size)

    def set_dtime(self, hi, lo):
        """set_dtime(), src/taylor_adaptive_batch.cpp:562-606: one (hi, lo) pair for every batch element, or one pair per
        element; checked (dtime_checks(), include/heyoka/detail/taylor_common.hpp:231-249) before the times are touched,
        then normalised."""
        n = self._batch_size
        if np.ndim(hi) == 0 and np.ndim(lo) == 0:
            hi, lo = np.full(n, float(hi)), np.full(n, float(lo))
        else:
            hi, lo = np.array(hi, dtype=np.float64).reshape(-1), np.array(lo, dtype=np.float64).reshape(-1)
            if hi.size != n or lo.size != n:
                raise ValueError("Invalid number of new times specified in a Taylor integrator in batch mode: the batch "
                                 "size is %d, but the number of specified times is (%d, %d)" % (n, hi.size, lo.size))
        for h, l in zip(hi.tolist(), lo.tolist()):
            if not (np.isfinite(h) and np.isfinite(l)):
                raise ValueError("The components of the double-length representation of the time coordinate must both "
                                 "be finite, but they are %r and %r instead" % (h, l))
            if abs(h) < abs(l):
                raise ValueError("The first component of the double-length representation of the time coordinate (%r) "
                                 "must not be smaller in magnitude than the second component (%r)" % (h, l))
        s = hi + lo
        self._t_lo = (hi - s) + lo
        self._t_hi = s

    @property
    def last_h(self):
        return self._last_h

    @property
    def step_res(self):
        return self._step_res

    @property
    def propagate_res(self):
        return self._prop_res

    @property
    def tc(self):
        return self._tc

    def get_decomposition_str(self):
        return self._prog.dc_str()

    # --- variational integrators (constructed from a var_ode_sys) ---------------------------------
    @property
    def is_variational(self):
        return self._vsys is not None

    @property
    def n_orig_sv(self):
        return self._prog.n_eq if self._vsys is None else self._vsys.n_orig_sv

    @property
    def vorder(self):
        return 0 if self._vsys is None else self._vsys.order

    @property
    def vargs(self):
        return [] if self._vsys is None else list(self._vsys.vargs)

    def _check_variational(self, what):
        if self._vsys is None:
            raise ValueError("The function %s can be invoked only on a variational integrator" % what)

    def get_vslice(self, order, component=None):
        """Rows of the state holding the derivatives of the given order (0: the original state variables), of all
        components or of one."""
        self._check_variational("get_vslice()")
        n, m = self._vsys.n_orig_sv, len(self._vsys.vargs)
        if order > self._vsys.order:
            raise ValueError("Cannot fetch the slice of the derivatives of order %d in a variational integrator of "
                             "order %d" % (order, self._vsys.order))
        if component is None:
            return slice(0, n) if order == 0 else slice(n, n * (1 + m))
        if not 0 <= component < n:
            raise ValueError("Cannot fetch the slice of the derivatives of the component %d in a variational "
                             "integrator with %d original state variables" % (component, n))
        return slice(component, component + 1) if order == 0 else slice(n + component * m, n + (component + 1) * m)

    def get_mindex(self, i):
        """Dense multi-index of state row i: [component, n_0, .., n_{m-1}]."""
        self._check_variational("get_mindex()")
        n, m = self._vsys.n_orig_sv, len(self._vsys.vargs)
        if not 0 <= i < n * (1 + m):
            raise ValueError("Cannot fetch the multi-index of the state variable %d in a variational integrator with "
                             "%d state variables" % (i, n * (1 + m)))
        if i < n:
            return [i] + [0] * m
        k = i - n
        return [k // m] + [1 if j == k % m else 0 for j in range(m)]

    def eval_taylor_map(self, dx):
        """Taylor map x + Phi dx of the current state, on the device: dx [n_args, batch]; returns tstate
        [n_orig_sv, batch]."""
        self._check_variational("eval_taylor_map()")
        m, n = len(self._vsys.vargs), self._batch_size
        dx = np.asarray(dx, dtype=np.float64)
        if dx.size != m * n:
            raise ValueError("Invalid number of values passed to eval_taylor_map(): %d values were passed, but %d are "
                             "needed (%d arguments in batches of %d)" % (dx.size, m * n, m, n))
        self._push()
        self._b.eval_taylor_map(self._vsys.n_orig_sv, dx.reshape(m, n), out=self._tstate)
        return self._tstate

    @property
    def tstate(self):
        return self._tstate

    # --- stepping ------------------------------------------------------------------------------
    def _push(self):
        self._b.upload(self._state, self._pars if self._prog.n_pars else None, self._t_hi, self._t_lo)

    def _pull(self, wtc):
        self._state, self._t_hi, self._t_lo, self._last_h = self._b.download()
        if wtc:
            self._tc = self._b.tc()

    def with_events(self):
        return self._with_events

    def get_t_events(self):
        if not self._with_events:
            raise ValueError("No events were defined for this integrator")  # src/taylor_adaptive_batch.cpp:2202-2229
        return self._tes

    def get_nt_events(self):
        if not self._with_events:
            raise ValueError("No events were defined for this integrator")
        return self._ntes

    def reset_cooldowns(self, i=None):
        if not self._with_events:
            raise ValueError("No events were defined for this integrator")
        self._b.reset_cooldowns(-1 if i is None else int(i))

    @property
    def te_cooldowns(self):
        """Cooldown state of the terminal events, [batch index][event index]: None = not in cooldown, else
        (time spent in cooldown, cooldown) (get_te_cooldowns(), src/taylor_adaptive_batch.cpp:2212-2219)."""
        if not self._with_events:
            raise ValueError("No events were defined for this integrator")
        n_te = len(self._tes)
        a, s, c = self._b.cooldowns(n_te)
        return [[(float(s[k, i]), float(c[k, i])) if a[k, i] else None for k in range(n_te)]
                for i in range(self._batch_size)]

    def _step_impl(self, max_delta_ts, backward, write_tc):
        self._push()
        self._b.step(max_delta_ts, backward=backward, write_tc=write_tc)
        # With events the Taylor coefficients are written unconditionally (src/taylor_adaptive_batch.cpp:776).
        self._pull(write_tc or self._with_events)
        oc, h = self._b.step_res()
        self._step_res = list(zip(oc.tolist(), h.tolist()))
        if self._with_events:
            self._run_event_callbacks()

    def _run_event_callbacks(self):
        """The callback part of the events branch of step_impl() (src/taylor_adaptive_batch.cpp:803-1033)."""
        evs = self._b.events()
        if not evs:
            return
        t_copy = (self._t_hi.copy(), self._t_lo.copy())
        excs = []
        lanes = sorted({e[0] for e in evs})
        for lane in lanes:
            mine = [e for e in evs if e[0] == lane]
            h = self._last_h[lane]
            thrown = False
            for (_, idx, terminal, d_sgn, t, _ad) in mine:
                if terminal:
                    continue
                # new_time - last_h + t in double-length arithmetic (:889).
                hi, lo = _dfloat_add(t_copy[0][lane], t_copy[1][lane], -h, 0.0)
                hi, lo = _dfloat_add(hi, lo, t, 0.0)
                try:
                    self._ntes[idx].callback(self, float(hi), d_sgn, lane)
                except Exception as e:  # noqa: BLE001 - collected and re-raised below like the reference
                    excs.append((lane, e))
                    thrown = True
                    break
            if thrown:
                continue
            te = [e for e in mine if e[2]]
            if te:
                _, idx, _, d_sgn, _t, _ad = te[0]
                ret = False
                cb = self._tes[idx].callback
                if cb is not None:
                    try:
                        ret = bool(cb(self, d_sgn, lane))
                    except Exception as e:  # noqa: BLE001
                        excs.append((lane, e))
                        continue
                self._step_res[lane] = (idx if ret else -idx - 1, self._step_res[lane][1])
        if len(excs) == 1:
            raise excs[0][1]
        if excs:
            msg = "Two or more exceptions were raised during the execution of event callbacks in a batch integrator:\n\n"
            for lane, e in excs:
                msg += "Batch index #%d:\n    Exception type: %s\n    Exception message: %s\n\n" % (
                    lane, type(e).__name__, e)
            raise RuntimeError(msg)
        same = lambda a, b: np.array_equal(a, b, equal_nan=True)  # noqa: E731
        if not (same(self._t_hi, t_copy[0]) and same(self._t_lo, t_copy[1])):
            i = int(np.argmax(~((self._t_hi == t_copy[0]) | (np.isnan(self._t_hi) & np.isnan(t_copy[0])))))
            raise RuntimeError("The invocation of one or more event callbacks resulted in the alteration of the time "
                               "coordinate of the integrator at the batch index %d - this is not supported" % i)

    def step(self, max_delta_ts=None, write_tc=False):
        if max_delta_ts is not None:
            m = np.asarray(max_delta_ts, dtype=np.float64)
            if m.size != self._batch_size:
                raise ValueError("Invalid number of max timesteps specified in a Taylor integrator in batch mode: the "
                                 "batch size is %d, but the number of specified timesteps is %d"
                                 % (self._batch_size, m.size))
            if np.any(np.isnan(m)):
                raise ValueError("Cannot use a nan max_delta_t in the step() function of an adaptive Taylor "
                                 "integrator in batch mode")
            max_delta_ts = m
        self._step_impl(max_delta_ts, False, write_tc)

    def step_backward(self, write_tc=False):
        self._step_impl(None, True, write_tc)

    def _propagate_until_host(self, th, tl, max_delta_t, max_steps, write_tc, callback, c_output=False):
        """The reference's lock-step loop (src/taylor_adaptive_batch.cpp:1256-1530) on the host, one device step per
        iteration: integrators with events (their callbacks are host code) and step callbacks."""
        n = self._batch_size
        tl = np.zeros(n) if tl is None else tl
        if not (np.all(np.isfinite(th)) and np.all(np.isfinite(tl))):
            raise ValueError("A non-finite time was passed to the propagate_until() function of an adaptive Taylor "
                             "integrator in batch mode")
        if max_delta_t is not None:
            if np.any(np.isnan(max_delta_t)):
                raise ValueError("A nan max_delta_t was passed to the propagate_until() function of an adaptive Taylor "
                                 "integrator in batch mode")
            if np.any(max_delta_t <= 0):
                raise ValueError("A non-positive max_delta_t was passed to the propagate_until() function of an "
                                 "adaptive Taylor integrator in batch mode")
        mdt = np.full(n, np.inf) if max_delta_t is None else np.asarray(max_delta_t, dtype=np.float64)
        rem_hi, rem_lo = _dfloat_add(th, tl, -self._t_hi, -self._t_lo)
        if not (np.all(np.isfinite(rem_hi)) and np.all(np.isfinite(rem_lo))):
            raise OverflowError("The final time passed to the propagate_until() function of an adaptive Taylor "
                                "integrator in batch mode results in an overflow condition")
        t_dir = (rem_hi > 0) | ((rem_hi == 0) & (rem_lo >= 0))
        self._prop_res = [(0, 0.0, 0.0, 0)] * n
        # Continuous output (integrators with events): the iterations of this loop are recorded on the device
        # (hy_cout_rec_*: update_c_out() / make_c_out(), src/taylor_adaptive_batch.cpp:1277-1346).
        rec = C.c_void_p()
        if c_output:
            self._push()
            check(lib.hy_cout_rec_begin(self._b._h, C.byref(rec)))

        def finish():
            if not rec.value:
                return None
            fwd = np.ascontiguousarray(t_dir, dtype=np.uint8)
            h, r = C.c_void_p(), C.c_void_p(rec.value)
            rec.value = None  # (finish destroys the recorder)
            check(lib.hy_cout_rec_finish(self._b._h, r, fwd.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(h)))
            return continuous_output_batch(h, self._prog.n_eq, n, self._prog.order) if h.value else None
        try:
            return self._propagate_until_host_loop(th, tl, mdt, rem_hi, rem_lo, t_dir, max_steps, write_tc, callback, rec,
                                                   finish)
        finally:
            if rec.value:
                lib.hy_cout_rec_destroy(rec)

    def _propagate_until_host_loop(self, th, tl, mdt, rem_hi, rem_lo, t_dir, max_steps, write_tc, callback, rec, finish):
        n = self._batch_size
        ts_count = [0] * n
        min_h, max_h = [float("inf")] * n, [0.0] * n
        iters = 0
        SUCCESS, STEP_LIMIT, NF, CB_STOP = _capi.HY_OUTCOME_SUCCESS, _capi.HY_OUTCOME_STEP_LIMIT, \
            _capi.HY_OUTCOME_ERR_NF_STATE, _capi.HY_OUTCOME_CB_STOP
        while True:
            cur = np.empty(n)
            for i in range(n):
                # min(dfloat(max_delta_t), rem) forward, max(dfloat(-max_delta_t), rem) backward, cast to double.
                if t_dir[i]:
                    cur[i] = mdt[i] if (mdt[i], 0.0) < (rem_hi[i], rem_lo[i]) else rem_hi[i]
                else:
                    cur[i] = rem_hi[i] if (-mdt[i], 0.0) < (rem_hi[i], rem_lo[i]) else -mdt[i]
            self._step_impl(cur, False, write_tc)
            n_done, nfs, ste = 0, False, False
            for i in range(n):
                oc, h = self._step_res[i]
                if oc == NF:
                    nfs = True
                else:
                    ts_count[i] += int(h != 0)
                    if oc == SUCCESS:
                        min_h[i], max_h[i] = min(min_h[i], abs(h)), max(max_h[i], abs(h))
                    ste = ste or (SUCCESS < oc < 0)
                    if h == rem_hi[i]:
                        n_done += 1
                        rem_hi[i] = rem_lo[i] = 0.0
                    else:
                        a, b = _dfloat_add(th[i], tl[i], -self._t_hi[i], -self._t_lo[i])
                        rem_hi[i], rem_lo[i] = float(a), float(b)
                self._prop_res[i] = (oc, min_h[i], max_h[i], ts_count[i])
            if nfs:
                return finish()
            if rec.value:
                check(lib.hy_cout_rec_append(self._b._h, rec))
            iters += 1
            if callback is not None:
                t_copy = (self._t_hi.copy(), self._t_lo.copy())
                ret = callback(self)
                if not (np.array_equal(self._t_hi, t_copy[0]) and np.array_equal(self._t_lo, t_copy[1])):
                    raise RuntimeError("The invocation of the callback passed to propagate_until() resulted in the "
                                       "alteration of the time coordinate of the integrator - this is not supported")
                if not ret:
                    self._prop_res = [(CB_STOP,) + r[1:] for r in self._prop_res]
                    return finish()
            if n_done == n or ste:
                return finish()
            if iters == max_steps:
                self._prop_res = [(STEP_LIMIT,) + r[1:] for r in self._prop_res]
                return finish()

    def propagate_until(self, ts, max_steps=0, max_delta_t=None, write_tc=False, callback=None, c_output=False):
        n = self._batch_size
        if np.ndim(ts) == 0:
            th, tl = np.full(n, float(ts)), None
        elif isinstance(ts, tuple):
            th, tl = np.asarray(ts[0], dtype=np.float64), np.asarray(ts[1], dtype=np.float64)
        else:
            th, tl = np.asarray(ts, dtype=np.float64), None
        if th.size != n:
            raise ValueError("Invalid number of time limits specified in a Taylor integrator in batch mode: the batch "
                             "size is %d, but the number of specified time limits is %d" % (n, th.size))
        if not (np.all(np.isfinite(self._t_hi)) and np.all(np.isfinite(self._t_lo))):
            raise ValueError("Cannot invoke the propagate_until() function of an adaptive Taylor integrator in batch "
                             "mode if one of the current times is not finite")
        if max_delta_t is not None:
            md = np.broadcast_to(np.asarray(max_delta_t, dtype=np.float64), (n,)) if np.ndim(max_delta_t) == 0 else \
                np.asarray(max_delta_t, dtype=np.float64)
            if md.size != n:
                raise ValueError("Invalid number of max timesteps specified in a Taylor integrator in batch mode: the "
                                 "batch size is %d, but the number of specified timesteps is %d" % (n, md.size))
            max_delta_t = md
        if self._with_events or (callback is not None and not c_output):
            return self._propagate_until_host(th, np.zeros(n) if tl is None else tl, max_delta_t, max_steps, write_tc,
                                              callback, c_output)
        self._push()
        c_out = None
        if c_output:
            # (The lock-step loop writes the Taylor coefficients at every iteration.)
            step_cb, err = None, []
            if callback is not None:
                # The step callback after every recorded iteration (src/taylor_adaptive_batch.cpp:1476-1500): the mirrors
                # are refreshed for it; it may alter state and parameters (uploaded again) but not the time.
                def step_cb():
                    try:
                        self._pull(True)
                        oc, mn, mx, ns = self._b.prop_res()
                        self._prop_res = list(zip(oc.tolist(), mn.tolist(), mx.tolist(), ns.tolist()))
                        t_copy = (self._t_hi.copy(), self._t_lo.copy())
                        go = callback(self)
                        if not (np.array_equal(self._t_hi, t_copy[0]) and np.array_equal(self._t_lo, t_copy[1])):
                            raise RuntimeError("The invocation of the callback passed to propagate_until() resulted in "
                                               "the alteration of the time coordinate of the integrator - this is not "
                                               "supported")
                        self._push()
                        return 1 if go else 0
                    except BaseException as e:  # noqa: BLE001 - carried across the C frame, re-raised below
                        err.append(e)
                        return -1
            c_out = self._b.propagate_until_cout(th, tl, max_delta_t, max_steps, step_cb=step_cb)
            if err:
                raise err[0]
            write_tc = True
        else:
            self._b.propagate_until(th, tl, max_delta_t, max_steps, write_tc)
        self._pull(write_tc)
        oc, mn, mx, ns = self._b.prop_res()
        self._prop_res = list(zip(oc.tolist(), mn.tolist(), mx.tolist(), ns.tolist()))
        return c_out

    def propagate_grid(self, grid, max_steps=0, max_delta_t=None, callback=None):
        """States at the grid points, shape [n_pts, n_eq, batch] (src/taylor_adaptive_batch.cpp:1545-2055).
        grid: [n_pts, batch] (or flat, point-major like the reference's std::vector)."""
        n = self._batch_size
        g = np.asarray(grid, dtype=np.float64).reshape(-1)
        if g.size == 0:
            raise ValueError("Cannot invoke propagate_grid() in an adaptive Taylor integrator in batch mode if the "
                             "time grid is empty")
        if g.size % n != 0:
            raise ValueError("Invalid grid size detected in propagate_grid() for an adaptive Taylor integrator in "
                             "batch mode: the grid has a size of %d, which is not a multiple of the batch size (%d)"
                             % (g.size, n))
        if max_delta_t is not None:
            md = np.broadcast_to(np.asarray(max_delta_t, dtype=np.float64), (n,)) if np.ndim(max_delta_t) == 0 else \
                np.asarray(max_delta_t, dtype=np.float64)
            if md.size != n:
                raise ValueError("Invalid number of max timesteps specified in a Taylor integrator in batch mode: the "
                                 "batch size is %d, but the number of specified timesteps is %d" % (n, md.size))
            max_delta_t = np.ascontiguousarray(md)
        if self._with_events or callback is not None or self._b.n_shards != 0:
            # (Host loop: events and step callbacks are host code; a batch sharded over several devices samples its grid
            # through the dense output of its shards.)
            return self._propagate_grid_host(g.reshape(-1, n), max_delta_t, max_steps, callback)
        self._push()
        out = self._b.propagate_grid(g.reshape(-1, n), max_delta_t, max_steps)
        self._pull(True)
        oc, mn, mx, ns = self._b.prop_res()
        self._prop_res = list(zip(oc.tolist(), mn.tolist(), mx.tolist(), ns.tolist()))
        return out

    def _propagate_grid_host(self, grid, max_delta_t, max_steps, callback):
        """propagate_grid() of an integrator with events / with a step callback: the reference's loop
        (src/taylor_adaptive_batch.cpp:1696-2053) on the host."""
        n, n_pts, dim = self._batch_size, grid.shape[0], self._prog.n_eq
        self._push()
        self._b.check_grid(grid, max_delta_t)
        out = np.full((n_pts, dim, n), np.nan)
        self.propagate_until(grid[0].copy(), max_steps=max_steps, max_delta_t=max_delta_t, write_tc=True)
        TO = taylor_outcome
        if any(r[0] != TO.time_limit for r in self._prop_res):
            self._prop_res = [(r[0], float("inf"), 0.0, 0) for r in self._prop_res]
            return out
        out[0] = self._state
        last = grid[n_pts - 1]
        rem_hi, rem_lo = _dfloat_add(last, np.zeros(n), -self._t_hi, -self._t_lo)
        if not (np.all(np.isfinite(rem_hi)) and np.all(np.isfinite(rem_lo))):
            raise ValueError("The final time passed to the propagate_grid() function of an adaptive Taylor integrator "
                             "in batch mode results in an overflow condition")
        t_dir = (rem_hi > 0) | ((rem_hi == 0) & (rem_lo >= 0))
        mdt = np.full(n, np.inf) if max_delta_t is None else max_delta_t
        ts_count, min_h, max_h = [0] * n, [float("inf")] * n, [0.0] * n
        cur = np.ones(n, dtype=np.int64)
        iters = 0
        if callback is not None and hasattr(callback, "pre_hook"):
            callback.pre_hook(self)
        while np.any(cur < n_pts):
            c_hi, c_lo = _dfloat_add(self._t_hi, self._t_lo, -self._last_h, np.zeros(n))
            pairs = [((self._t_hi[i], self._t_lo[i]), (c_hi[i], c_lo[i])) for i in range(n)]
            t0, t1 = [min(p) for p in pairs], [max(p) for p in pairs]
            dflags = np.ones(n, dtype=bool)
            while True:
                pg = np.zeros(n)
                for i in range(n):
                    if dflags[i] and cur[i] < n_pts:
                        g = grid[cur[i], i]
                        dflags[i] = (t0[i] <= (g, 0.0) <= t1[i]) or (rem_hi[i] == 0 and rem_lo[i] == 0)
                        pg[i] = g
                    else:
                        dflags[i] = False
                if not dflags.any():
                    break
                d = self.update_d_output(pg)
                for i in np.nonzero(dflags)[0]:
                    out[cur[i], :, i] = d[:, i]
                    cur[i] += 1
                if not np.any(cur < n_pts):
                    break
            if not np.any(cur < n_pts):
                break
            if any(r[0] in (TO.cb_stop, TO.step_limit) or TO.success < r[0] < 0 for r in self._prop_res):
                break
            lim = np.empty(n)
            for i in range(n):
                if t_dir[i]:
                    lim[i] = mdt[i] if (mdt[i], 0.0) < (rem_hi[i], rem_lo[i]) else rem_hi[i]
                else:
                    lim[i] = rem_hi[i] if (-mdt[i], 0.0) < (rem_hi[i], rem_lo[i]) else -mdt[i]
            self._step_impl(lim, False, True)
            nfs = False
            for i in range(n):
                oc, h = self._step_res[i]
                if oc == TO.err_nf_state:
                    nfs = True
                else:
                    ts_count[i] += int(h != 0)
                    if oc == TO.success:
                        min_h[i], max_h[i] = min(min_h[i], abs(h)), max(max_h[i], abs(h))
                    if h == rem_hi[i]:
                        rem_hi[i] = rem_lo[i] = 0.0
                    else:
                        a, b = _dfloat_add(last[i], 0.0, -self._t_hi[i], -self._t_lo[i])
                        rem_hi[i], rem_lo[i] = float(a), float(b)
                self._prop_res[i] = (oc, min_h[i], max_h[i], ts_count[i])
            if nfs:
                break
            iters += 1
            if callback is not None:
                t_copy = (self._t_hi.copy(), self._t_lo.copy())
                ret = callback(self)
                if not (np.array_equal(self._t_hi, t_copy[0]) and np.array_equal(self._t_lo, t_copy[1])):
                    raise RuntimeError("The invocation of the callback passed to propagate_grid() resulted in the "
                                       "alteration of the time coordinate of the integrator - this is not supported")
                if not ret:
                    self._prop_res = [(TO.cb_stop,) + r[1:] for r in self._prop_res]
                    continue
            if iters == max_steps:
                self._prop_res = [(TO.step_limit,) + r[1:] for r in self._prop_res]
        return out

    def propagate_for(self, delta_ts, **kw):
        n = self._batch_size
        d = np.broadcast_to(np.asarray(delta_ts, dtype=np.float64), (n,)) if np.ndim(delta_ts) == 0 else \
            np.asarray(delta_ts, dtype=np.float64)
        if d.size != n:
            raise ValueError("Invalid number of time intervals specified in a Taylor integrator in batch mode: the "
                             "batch size is %d, but the number of specified time intervals is %d" % (n, d.size))
        hi, lo = _dfloat_add(self._t_hi, self._t_lo, d, np.zeros(n))
        return self.propagate_until((hi, lo), **kw)

    def update_d_output(self, t, rel_time=False):
        """Dense output at time(s) t from the last written tc (src/taylor_adaptive_batch.cpp:2251-2327)."""
        n = self._batch_size
        t = np.broadcast_to(np.asarray(t, dtype=np.float64), (n,))
        if rel_time:
            # Relative to the CURRENT time; the polynomial is expanded about the start of the last step (:2276-2280).
            tau = self._last_h + t
        else:
            # tau = t - (time - last_h), in double-length arithmetic.
            hi, lo = _dfloat_add(self._t_hi, self._t_lo, -self._last_h, np.zeros(n))
            tau, _ = _dfloat_add(t, np.zeros(n), -hi, -lo)
        return self._b.d_output(tau)


def _var_initial_state(vsys, state, batch):
    """The constructor's fill of the variational rows (taylor.hpp): original rows as given (zeros if the state is
    empty); per lane, the STM column of an argument that is the state variable x_k is e_k, that of a parameter 0."""
    n, m = vsys.n_orig_sv, len(vsys.vargs)
    full = np.zeros((n * (1 + m), batch))
    if state.size:
        full[:n] = state.reshape(n, batch)
    for i in range(n):
        for j, a in enumerate(vsys.vargs):
            if repr(diff(a, vsys.sys[i][0])) == "1":  # a is the state variable x_i (a parameter gives 0)
                full[n + i * m + j] = 1.0
    return full


def _eft_knuth(a, b):
    x = a + b
    z = x - a
    y = (a - (x - z)) + (b - z)
    return x, y


def _eft_dekker(a, b):
    x = a + b
    y = (a - x) + b
    return x, y


def _dfloat_add(ahi, alo, bhi, blo):
    """include/heyoka/detail/dfloat.hpp:151-169."""
    xh, yh = _eft_knuth(ahi, bhi)
    xl, yl = _eft_knuth(alo, blo)
    u, v = _eft_dekker(xh, yh + xl)
    u, v = _eft_dekker(u, v + yl)
    return u, v
