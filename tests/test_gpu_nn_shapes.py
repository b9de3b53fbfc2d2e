"""The dense-network kernel (k_nn, heyoka_b200/csrc/nn_kernel.cuh) over network shapes: the planner (nn_plan.cpp) and
setup_nn() (batch.cu) restated on the CPU, the device's Taylor coefficients against a 50-digit series reference of the
network, and the device bit for bit against k_hbm where the arithmetic says it must be.

Why not bit for bit everywhere. A dense layer is one matrix product on the FP64 tensor cores (DMMA), which sums a
neuron's products in another association than the reference's nested 8-term sums (nn_kernel.cuh, DESIGN.md 4.8). So
dense networks are compared with the series reference under NN_BOUND, calibrated on the CPU oracle in its three
summation modes. Bit equality is asserted where it follows from the arithmetic: networks in which every neuron has
exactly one product (DMMA then adds exact zeros to one rounded product), lanes of k_nn against the same lanes run alone,
and a sharded batch against a single-device one.

The case matrix (CASES) is chosen so that every path of the kernel's layer loop runs: full tiles, the second DMMA chain
of the generic k-loop, masked k, partial tiles, more than one tile per warp, more (neuron, lane) items than threads, one
TMA chunk and several, and a program past the shared-memory fit. test_every_path_is_reached() derives from the widths,
without a GPU, which case reaches which path.

NN_BOUND = 5e-12. Calibration (test_oracle_meets_nn_bound, x86-64): the oracle's worst normalised error over every case,
order and summation mode is 5.5e-13 (3:[130]; every other case stays below 2.3e-13), so the bound is about 9 times
above it. On an H100 (700 W) k_nn's worst is 6.0e-13, also on 3:[130]. The normalisation is per state variable and
order, with no |h|^o weight: the high orders of a tanh network are sums that cancel, and a relative error of 1e-13 there
is the reference's own. A coefficient of the wrong order, lane or neuron moves the error by O(1)."""
import ctypes as C
import functools
import os
import re
import subprocess

import numpy as np
import pytest

import heyoka_b200 as hb
import oracle
import series_ref as sr
from test_gpu_parity import lane_err

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "heyoka_b200", "csrc")
LIBDIR = os.path.join(ROOT, "heyoka_b200", "lib")
SO = os.path.join(ROOT, "build", "libnn_emul.so")

SMEM_OPTIN = 227 * 1024  # cudaDeviceProp::sharedMemPerBlockOptin of an H100
H100_SMS = 132
NN_LB = 2                # lanes per CTA (nn_kernel.cuh)
NN_THREADS = 256
TMA_CHUNK = 32768        # bytes per cp.async.bulk of the weight image
NN_BOUND = 5e-12
NF = hb.taylor_outcome.err_nf_state
EPS = np.finfo(np.float64).eps


# ---- the planner, called through tests/cpp/nn_emul.cpp --------------------------------------------------------------

@functools.cache
def _emul():
    src = os.path.join(ROOT, "tests", "cpp", "nn_emul.cpp")
    deps = [src, os.path.join(CSRC, "nn_plan.hpp"), os.path.join(CSRC, "nn_plan.cpp"), os.path.join(CSRC, "program.hpp"),
            os.path.join(LIBDIR, "libheyoka_b200.so")]
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    if not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(d) for d in deps):
        # (Built under a private name and renamed: the case matrix plans its networks when the file is collected, which
        # several test processes may do at once.)
        tmp = "%s.%d" % (SO, os.getpid())
        subprocess.run(["g++", "-std=c++17", "-O2", "-shared", "-fPIC", "-I" + os.path.join(ROOT, "include"), "-I" + CSRC,
                        src, "-o", tmp, "-L" + LIBDIR, "-lheyoka_b200", "-Wl,-rpath," + LIBDIR], check=True)
        os.replace(tmp, SO)
    lib = C.CDLL(SO)
    lib.nn_emul_plan.restype = C.c_int
    return lib


def nn_emul_plan(P):
    """make_nn_plan() of a program: dict(ok, why, layers = [dict(n_in, n_out, act, w [n_out, n_in], bias)], out_of_sv)."""
    lib = _emul()
    info = (C.c_uint32 * 26)()
    why = C.create_string_buffer(256)
    oos = np.zeros(P.n_eq, dtype=np.uint32)
    dp = C.POINTER(C.c_double)
    assert lib.nn_emul_plan(P._h, info, why, C.c_size_t(256), oos.ctypes.data_as(C.POINTER(C.c_uint32)), None,
                            C.c_size_t(0), None, C.c_size_t(0)) == 0
    out = dict(ok=bool(info[0]), why=why.value.decode(), layers=[], out_of_sv=oos)
    if not out["ok"]:
        return out
    dims = [(info[2 + 3 * l], info[3 + 3 * l], info[4 + 3 * l]) for l in range(info[1])]
    w = np.zeros(sum(i * o for i, o, _ in dims))
    b = np.zeros(sum(o for _, o, _ in dims))
    assert lib.nn_emul_plan(P._h, info, why, C.c_size_t(256), oos.ctypes.data_as(C.POINTER(C.c_uint32)),
                            w.ctypes.data_as(dp), C.c_size_t(w.size), b.ctypes.data_as(dp), C.c_size_t(b.size)) == 0
    wo = bo = 0
    for n_in, n_out, act in dims:
        out["layers"].append(dict(n_in=n_in, n_out=n_out, act=act, w=w[wo:wo + n_in * n_out].reshape(n_out, n_in),
                                  bias=b[bo:bo + n_out]))
        wo, bo = wo + n_in * n_out, bo + n_out
    return out


# ---- setup_nn(), restated ------------------------------------------------------------------------------------------

def nn_expected(plan, n_eq, order, batch):
    """What setup_nn() (batch.cu) lays out for a planned network on an H100: the weight image (rows padded to
    n_in_pad = 4k and then to ldw = 4 mod 16 doubles, n_out_pad = 8k rows, each bias block padded to an even count),
    the histories (z, tanh, tanh^2: 3 order n_out LB doubles per hidden layer), the state-variable coefficients, the
    output buffer and the scalars; the fit test bytes + 2048 <= 227 KB; grid = min(132, ceil(batch / 2)). None if the
    planner refused the program."""
    if not plan["ok"] or len(plan["layers"]) > 8:
        return None
    img = hist = max_out = 0
    layers = []
    for L in plan["layers"]:
        n_in_pad, n_out_pad = (L["n_in"] + 3) & ~3, (L["n_out"] + 7) & ~7
        ldw = n_in_pad
        while ldw % 16 != 4:
            ldw += 1
        img += n_out_pad * ldw
        img = (img + L["n_out"] + 1) & ~1
        if L["act"] != 0:
            hist += 3 * order * L["n_out"] * NN_LB
        max_out = max(max_out, L["n_out"])
        layers.append(dict(L, n_in_pad=n_in_pad, n_out_pad=n_out_pad, ldw=ldw))
    doubles = img + hist + (order + 1) * n_eq * NN_LB + max_out * NN_LB + NN_LB + 4
    return dict(tape="nn", smem_bytes=doubles * 8, grid=max(1, min(H100_SMS, -(-batch // NN_LB))),
                fits=doubles * 8 + 2048 <= SMEM_OPTIN, wimg_bytes=img * 8, layers=layers)


def nn_paths(e, n_eq):
    """The paths of k_nn's jet that a layout reaches (nn_kernel.cuh, the layer loop of jet())."""
    out = set()
    for L in e["layers"]:
        kpad = L["n_in_pad"]
        if L["n_in"] == kpad and kpad % 8 == 0:
            out.add("full tile")
        else:
            if kpad > 4:
                out.add("second chain")          # k0 + 4 < kpad at k0 = 0
            if kpad % 8 == 4 and kpad > 4:
                out.add("second chain skipped")  # ... and not at the last k0
            if L["n_in"] % 4 != 0:
                out.add("masked k")
        if L["act"] != 0 and L["n_out"] % 8 != 0:
            out.add("partial hidden tile")
        if L["n_out_pad"] > 8 * NN_THREADS // 32:
            out.add("tiles per warp > 1")
        if L["act"] != 0 and L["n_out"] * NN_LB > NN_THREADS:
            out.add("items > threads")
    out.add("one TMA chunk" if e["wimg_bytes"] <= TMA_CHUNK else "several TMA chunks")
    out.add("fits" if e["fits"] else "does not fit")
    if len(e["layers"]) == 1:
        out.add("linear only")
    if len(e["layers"]) == 8:
        out.add("maximum depth")
    return out


ALL_PATHS = {"full tile", "second chain", "second chain skipped", "masked k", "partial hidden tile", "tiles per warp > 1",
             "items > threads", "one TMA chunk", "several TMA chunks", "fits", "does not fit", "linear only",
             "maximum depth", "out_of_sv not the identity"}


# ---- the networks --------------------------------------------------------------------------------------------------

def _net_weights(n_eq, hidden, seed, one_product=False, sparse=False):
    """[(W [n_out, n_in], b)] of a network n_eq -> hidden -> n_eq: W ~ N(0, 1 / fan_in), b ~ N(0, 0.1) as in
    common.sys_ffnn(). one_product: every neuron reads exactly one input, input (perm[i] mod n_in) of a random
    permutation, with a weight of at least 0.5 in magnitude and a non-zero bias. sparse: weights drawn from {0, +1, -1,
    N(0, 1 / fan_in)}, every row and column with a non-zero."""
    rng = np.random.default_rng(seed)
    sizes = [n_eq] + list(hidden) + [n_eq]
    out = []
    for n_in, n_out in zip(sizes[:-1], sizes[1:]):
        if one_product:
            W = np.zeros((n_out, n_in))
            perm = rng.permutation(max(n_in, n_out))
            for i in range(n_out):
                W[i, perm[i] % n_in] = rng.choice([-1., 1.]) * rng.uniform(0.5, 1.5)
        elif sparse:
            W = rng.normal(0, 1 / np.sqrt(n_in), (n_out, n_in))
            kind = rng.integers(0, 4, (n_out, n_in))
            W[kind == 0], W[kind == 1], W[kind == 2] = 0., 1., -1.
            for i in range(n_out):
                if not W[i].any():
                    W[i, rng.integers(n_in)] = 1.
            for j in range(n_in):
                if not W[:, j].any():
                    W[rng.integers(n_out), j] = -1.
        else:
            W = rng.normal(0, 1 / np.sqrt(n_in), (n_out, n_in))
        b = rng.normal(0, 0.1, n_out)
        b[b == 0.] = 0.05
        out.append((W, b))
    return out


class Net:
    """A network x' = ffnn(x) built with hb.model.ffnn(): `outs[s]` is the output neuron that state variable s derives
    from. acts: the activations of the hidden layers (tanh by default; the output layer is linear)."""

    def __init__(self, name, n_eq, hidden, seed=0, outs=None, acts=None, one_product=False, sparse=False):
        self.name, self.n_eq, self.hidden = name, n_eq, list(hidden)
        self.outs = list(range(n_eq)) if outs is None else list(outs)
        self.acts = ["tanh"] * len(hidden) if acts is None else list(acts)
        self.wb = _net_weights(n_eq, hidden, seed, one_product=one_product, sparse=sparse)

    def nn_wb(self):
        return np.concatenate([W.reshape(-1) for W, _ in self.wb] + [b for _, b in self.wb])

    def sys(self):
        xs = hb.make_vars(*["x%d" % i for i in range(self.n_eq)])
        out = hb.model.ffnn(list(xs), self.hidden, self.n_eq, self.acts + ["identity"], nn_wb=self.nn_wb())
        return [(xs[s], out[self.outs[s]]) for s in range(self.n_eq)]

    def program(self, order):
        P = hb.Program(self.sys(), tol=sr.order_tol(order))
        assert P.order == order, (self.name, order, P.order)
        return P

    def states(self, batch, seed=1):
        """U(-1, 1), different in every lane."""
        return np.random.default_rng(seed).uniform(-1., 1., (self.n_eq, batch))

    def expected_plan(self):
        """The layers the planner must rebuild: the hidden layers as built, the output layer with the neurons that some
        state variable reads, numbered in the order the state variables first read them."""
        used = list(dict.fromkeys(self.outs))
        layers = [dict(w=W, bias=b, act=1) for W, b in self.wb[:-1]]
        W, b = self.wb[-1]
        layers.append(dict(w=W[used], bias=b[used], act=0))
        return layers, np.array([used.index(o) for o in self.outs], dtype=np.uint32)


def _cases():
    c = [Net("1:[3]", 1, [3], seed=1), Net("3:[13]", 3, [13], seed=2), Net("5:[12,12]", 5, [12, 12], seed=3),
         Net("4:[72]", 4, [72], seed=4), Net("3:[130]", 3, [130], seed=5), Net("8:[100,37]", 8, [100, 37], seed=6),
         Net("4:[]", 4, [], seed=7), Net("3:[9]*7", 3, [9] * 7, seed=8), Net("4:[64,64,64]", 4, [64, 64, 64], seed=9),
         # Output permutations: the planner numbers the output neurons in the order the state variables first read
         # them, so a permutation gives permuted rows and two state variables reading one neuron give out_of_sv [0, 0, 1].
         Net("3:[13]-perm", 3, [13], seed=10, outs=[2, 0, 1]), Net("3:[13]-shared", 3, [13], seed=11, outs=[0, 0, 2]),
         # Weights 0, +1 and -1: dropped products, plain inputs, negations and differences in the decomposition.
         Net("3:[13,9]-sparse", 3, [13, 9], seed=21, sparse=True)]
    return {n.name: n for n in c}


CASES = _cases()
NARROW = ("1:[3]", "3:[13]", "5:[12,12]", "4:[]", "3:[9]*7", "3:[13]-perm", "3:[13]-shared", "3:[13,9]-sparse")
ORDERS = (3, 8, 15, 20)
REF_LANES = 3


@functools.cache
def fit_boundary(name):
    """(the highest order at which case `name` fits in shared memory, the next one), from nn_expected()."""
    net = CASES[name]
    plan = nn_emul_plan(net.program(8))
    fits = [o for o in range(2, 120) if nn_expected(plan, net.n_eq, o, 1)["fits"]]
    assert fits == list(range(2, max(fits) + 1))
    return max(fits), max(fits) + 1


def _orders(name):
    out = list(ORDERS) + ([33] if name in NARROW else [])
    if name in ("3:[130]", "4:[64,64,64]"):
        out += list(fit_boundary(name))
    return sorted(set(out))


DENSE = [(name, o) for name in CASES for o in _orders(name)]


# ---- the series reference ------------------------------------------------------------------------------------------

def nn_series_jet(wb, acts, outs, x0, order):
    """The jet [n_eq][order + 1] (mpf, 50 digits) of x' = ffnn(x) from x0, for one lane: at every order n the layers are
    evaluated on the order-n coefficients of their inputs, z^[n] = W a^[n] (+ b at n = 0), and tanh as the quotient
    (e - 1) / (e + 1) of e = exp(2 z) (series_ref.s_tanh), both series extended by one term per order (e by its
    recurrence k e^[k] = sum_j 2 j z^[j] e^[k-j], the quotient by long division). Every z^[n], e^[n] and tanh^[n] is
    computed once: O(order^2) per neuron instead of O(order^3) for s_tanh() on the whole series at every order."""
    mpf, fsum = sr.mpf, sr.mp.fsum
    W = [[[mpf(float(v)) for v in row] for row in Wl] for Wl, _ in wb]
    B = [[mpf(float(v)) for v in bl] for _, bl in wb]
    acts = list(acts) + ["identity"]
    X = [[mpf(float(v))] for v in x0]
    Z = [[[] for _ in Bl] for Bl in B]  # per layer and neuron: z, e = exp(2 z), t = tanh(z)
    E = [[[] for _ in Bl] for Bl in B]
    T = [[[] for _ in Bl] for Bl in B]
    for n in range(order):
        a = [x[n] for x in X]
        for l in range(len(W)):
            z = [fsum(w * v for w, v in zip(row, a)) + (B[l][i] if n == 0 else 0) for i, row in enumerate(W[l])]
            if acts[l] != "tanh":
                a = z
                continue
            a = []
            for i, zi in enumerate(z):
                zs, es, ts = Z[l][i], E[l][i], T[l][i]
                zs.append(zi)
                if n == 0:
                    es.append(sr.mp.exp(2 * zi))
                    ts.append((es[0] - 1) / (es[0] + 1))
                else:
                    es.append(fsum(2 * j * zs[j] * es[n - j] for j in range(1, n + 1)) / n)
                    ts.append((es[n] - fsum(ts[n - j] * es[j] for j in range(1, n + 1))) / (es[0] + 1))
                a.append(ts[n])
        for s in range(len(X)):
            X[s].append(a[outs[s]] / (n + 1))
    return X


@functools.cache
def reference(name, order):
    """(states [n_eq, REF_LANES], float64 reference jets [n_eq, order + 1, REF_LANES]) of case `name`."""
    net = CASES[name]
    st = net.states(REF_LANES, seed=order)
    lanes = [nn_series_jet(net.wb, net.acts, net.outs, st[:, i], order) for i in range(REF_LANES)]
    ref = np.array([[[float(lanes[b][v][o]) for b in range(REF_LANES)] for o in range(order + 1)]
                    for v in range(net.n_eq)])
    return st, ref


# ---- CPU: the planner, setup_nn() and the reference ----------------------------------------------------------------

def plan_matches(plan, layers, oos):
    """The planner's layers are `layers` (dicts w, bias, act as built), bit for bit, up to the order in which it numbers
    the hidden neurons (the order of their tanh in the decomposition): the permutation that matches a layer's rows
    must be the one that matches the next layer's columns. Returns the permutations."""
    assert len(plan["layers"]) == len(layers)
    prev = np.arange(layers[0]["w"].shape[1])  # layer 0 reads the state variables in order
    perms = []
    for l, (got, exp) in enumerate(zip(plan["layers"], layers)):
        assert got["act"] == exp["act"] and got["w"].shape == exp["w"].shape, l
        w = exp["w"][:, prev]
        if exp["act"] == 0:
            perm = np.arange(w.shape[0])
        else:
            rows = {(w[i].tobytes(), exp["bias"][i].tobytes()): i for i in range(w.shape[0])}
            assert len(rows) == w.shape[0]
            perm = np.array([rows.get((got["w"][r].tobytes(), got["bias"][r].tobytes()), -1)
                             for r in range(w.shape[0])])
            assert sorted(perm) == list(range(w.shape[0])), (l, perm)
        assert np.array_equal(got["w"], w[perm]) and np.array_equal(got["bias"], exp["bias"][perm]), l
        perms.append(perm)
        prev = perm
    assert np.array_equal(plan["out_of_sv"], oos), plan["out_of_sv"]
    return perms


@pytest.mark.parametrize("name", list(CASES))
def test_planner_rebuilds_the_weights(name):
    """The matrices and biases make_nn_plan() walks back out of the decomposition are the nn_wb blocks, bit for bit
    (hidden neurons in the planner's order), and out_of_sv is the map that was built."""
    net = CASES[name]
    plan = nn_emul_plan(net.program(8))
    assert plan["ok"], plan["why"]
    plan_matches(plan, *net.expected_plan())


def test_planner_sparse_weights():
    """Weights 0, +1 and -1 with non-zero biases: the expression builder drops the zero products and folds the others
    into plain inputs, negations and differences (x - y, b - x), which the planner takes apart (the VAR, NEG, MUL_NV and
    SUB branches of expand()); it rebuilds the matrices bit for bit, zeros included. (Before the SUB branches existed
    such a network was refused, "a neuron contains opcode 4", and ran on a generic kernel.)"""
    net = CASES["3:[13,9]-sparse"]
    W0 = net.wb[0][0]
    assert (W0 == 0).any() and (W0 == 1).any() and (W0 == -1).any()
    P = net.program(8)
    ops = {sr.OPNAMES[op[0]] for op in P.ops_array()}
    assert {"MUL_NV", "SUB_VV", "SUB_NV"} <= ops, ops
    plan = nn_emul_plan(P)
    assert plan["ok"], plan["why"]
    plan_matches(plan, *net.expected_plan())


def test_planner_folds_identity_layers():
    """A hidden layer without activation is folded into the next one: expand() multiplies the weights through, so the
    planner's matrix is W2 W1 and its bias W2 b1 + b2. This is a reassociation across layers (each entry a sum of
    n_mid rounded products), so the bound is the one of a dot product, gamma_(n_mid + 1) (|W2| |W1|) elementwise."""
    net = Net("identity", 3, [7, 11, 5], seed=22, acts=["tanh", "identity", "tanh"])
    plan = nn_emul_plan(net.program(8))
    assert plan["ok"], plan["why"]
    assert [(L["n_in"], L["n_out"], L["act"]) for L in plan["layers"]] == [(3, 7, 1), (7, 5, 1), (5, 3, 0)]
    (W0, b0), (W1, b1), (W2, b2), (W3, b3) = net.wb
    # Layers 0 and 2 (the output layer) exactly; the neurons of each hidden layer in the planner's order.
    p0 = plan_matches(dict(plan, layers=plan["layers"][:1]), [dict(w=W0, bias=b0, act=1)], plan["out_of_sv"])[0]
    k = W1.shape[0] + 1
    gamma = k * EPS / 2 / (1 - k * EPS / 2)
    got, M, Mb = plan["layers"][1], (W2 @ W1)[:, p0], W2 @ b1 + b2
    bound, bound_b = gamma * (np.abs(W2) @ np.abs(W1))[:, p0], gamma * (np.abs(W2) @ np.abs(b1) + np.abs(b2))
    p1 = [int(np.argmin(np.max(np.abs(M - r), axis=1))) for r in got["w"]]
    assert sorted(p1) == list(range(M.shape[0]))
    assert np.all(np.abs(got["w"] - M[p1]) <= bound[p1]) and np.all(np.abs(got["bias"] - Mb[p1]) <= bound_b[p1])
    assert np.array_equal(plan["layers"][2]["w"], W3[:, p1]) and np.array_equal(plan["layers"][2]["bias"], b3)


def _hand_net(xs, W, b, extra=None):
    """tanh(W x + b) -> one linear output per state variable, built term by term like model::ffnn; extra(i) adds a
    term to the sum of hidden neuron i (None: nothing)."""
    hid = []
    for i in range(W.shape[0]):
        terms = [float(W[i, j]) * xs[j] for j in range(len(xs))] + [float(b[i])]
        if extra is not None:
            terms.append(extra(i))
        hid.append(hb.tanh(hb.sum(terms)))
    return hid


def refusals():
    """(name, system, the planner's reason)."""
    out = []
    net = Net("r", 3, [5], seed=23)
    for act in ("sigmoid", "relu", "sin", "exp"):
        n = Net("r-" + act, 3, [5], seed=23, acts=[act])
        out.append((act + " hidden layer", n.sys(), "a neuron contains opcode"))
    xs = hb.make_vars("x0", "x1", "x2")
    o = hb.model.ffnn(list(xs), [5], 3, ["tanh", "tanh"], nn_wb=net.nn_wb())
    out.append(("tanh output layer", [(xs[i], o[i]) for i in range(3)], "a state variable's derivative is not an output neuron"))
    deep = Net("r-deep", 3, [4] * 8, seed=24)
    out.append(("8 hidden layers", deep.sys(), "unsupported depth"))
    (W, b), (W2, b2) = net.wb
    hid = _hand_net(list(xs), W, b, extra=lambda i: hb.par[0] * xs[0] if i == 2 else 0.)
    out.append(("parameter in a weight", [(xs[s], hb.sum([float(W2[s, j]) * hid[j] for j in range(5)] + [float(b2[s])]))
                                          for s in range(3)], "no operations / runtime parameters"))
    hid = _hand_net(list(xs), W, b, extra=lambda i: 0.5 * hb.time if i == 1 else 0.)
    out.append(("time-dependent", [(xs[s], hb.sum([float(W2[s, j]) * hid[j] for j in range(5)] + [float(b2[s])]))
                                   for s in range(3)], "a neuron contains opcode"))
    hid = _hand_net(list(xs), W, b)
    out.append(("output reads a state variable", [(xs[s], hb.sum([float(W2[s, j]) * hid[j] for j in range(5)]
                                                                 + [float(b2[s])] + ([0.25 * xs[1]] if s == 0 else [])))
                                                  for s in range(3)], "a neuron reads something else than the previous layer"))
    return out


REFUSALS = [r[0] for r in refusals()]


@pytest.mark.parametrize("idx", range(len(REFUSALS)), ids=REFUSALS)
def test_planner_refusals(idx):
    name, sys_, why = refusals()[idx]
    plan = nn_emul_plan(hb.Program(sys_, tol=sr.order_tol(8)))
    assert not plan["ok"] and why in plan["why"], (name, plan["why"])


def test_every_path_is_reached():
    """(No GPU needed.) The dense cases of this file, at their orders, reach every path of k_nn's layer loop that
    nn_paths() names; the one-product cases do too, apart from the fit boundary."""
    seen = set()
    for name, order in DENSE:
        net = CASES[name]
        plan = nn_emul_plan(net.program(8))
        e = nn_expected(plan, net.n_eq, order, REF_LANES)
        seen |= nn_paths(e, net.n_eq)
        if not np.array_equal(plan["out_of_sv"], np.arange(net.n_eq)):
            seen.add("out_of_sv not the identity")
    assert seen == ALL_PATHS, ALL_PATHS - seen
    # The fit boundary is the one of setup_nn(): one order fits, the next does not.
    for name in ("3:[130]", "4:[64,64,64]"):
        lo, hi = fit_boundary(name)
        plan = nn_emul_plan(CASES[name].program(8))
        assert nn_expected(plan, CASES[name].n_eq, lo, 1)["fits"] and not nn_expected(plan, CASES[name].n_eq, hi, 1)["fits"]
    seen = set()
    for name in ONE_PRODUCT:
        net = ONE_PRODUCT[name]
        plan = nn_emul_plan(net.program(op_order(name)))
        assert plan["ok"], plan["why"]
        assert [L["n_out"] for L in plan["layers"]] == net.hidden + [net.n_eq]
        assert op_order(name) >= 8
        seen |= nn_paths(nn_expected(plan, net.n_eq, op_order(name), OP_BATCH), net.n_eq)
    assert seen >= ALL_PATHS - {"does not fit", "out_of_sv not the identity", "items > threads"}, ALL_PATHS - seen


def test_incremental_tanh_equals_s_tanh():
    """nn_series_jet()'s incremental tanh against series_ref.s_tanh() on the whole series: one neuron, x' = tanh(w x +
    b), whose jet is also series_ref.series_jet() of that right-hand side."""
    wb = [(np.array([[0.7]]), np.array([0.2])), (np.array([[1.3]]), np.array([-0.1]))]
    got = nn_series_jet(wb, ["tanh"], [0], [0.4], 12)
    ref = sr.series_jet(lambda m, x: [1.3 * m.tanh(0.7 * x[0] + 0.2) - 0.1], [0.4], [], 0., 12)
    assert all(abs(a - b) < 1e-45 for a, b in zip(got[0], ref[0]))


MODES = {"pairwise": oracle.PAIRWISE, "seq": oracle.SEQ, "fma": oracle.FMA}


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_meets_nn_bound(name):
    """The calibration of NN_BOUND: the oracle's jets in its three summation modes against the series reference, every
    coefficient normalised per variable and order (series_ref.normalised_err)."""
    worst = 0.
    for order in _orders(name):
        st, ref = reference(name, order)
        P = CASES[name].program(order)
        for mode in MODES.values():
            o = oracle.OracleIntegrator(P, st, REF_LANES, mode=mode)
            o.step(write_tc=True)
            err = sr.normalised_err(o.tc, ref)
            worst = max(worst, err)
            assert err < NN_BOUND, (name, order, mode, err)
    print("%s: oracle's worst normalised error %.3g" % (name, worst))


# ---- one-product networks ------------------------------------------------------------------------------------------
# Every neuron has exactly one non-zero weight. A neuron that nothing reads is not part of the decomposition, so every
# layer is at least as wide as the one before it and n_eq at least the widest (the output layer reads n_eq neurons):
# the widths of CASES with n_eq raised. The weight image keeps the zeros, so the widest networks of CASES do not fit as
# square layers: 8:[100, 37] becomes 44:[37, 44] (second chain skipped at the last k, masked k), 4:[64, 64, 64] loses
# a layer, and 3:[130] (items > threads) has no one-product counterpart that fits.

ONE_PRODUCT = {n.name: n for n in (
    Net("op 3:[3]", 3, [3], seed=31, one_product=True), Net("op 13:[13]", 13, [13], seed=32, one_product=True),
    Net("op 12:[12,12]", 12, [12, 12], seed=33, one_product=True), Net("op 72:[72]", 72, [72], seed=34, one_product=True),
    Net("op 44:[37,44]", 44, [37, 44], seed=36, one_product=True),
    Net("op 4:[]", 4, [], seed=37, one_product=True), Net("op 9:[9]*7", 9, [9] * 7, seed=38, one_product=True),
    Net("op 64:[64,64]", 64, [64, 64], seed=39, one_product=True))}


@functools.cache
def op_order(name):
    """Order 15, or the highest order below it at which the network fits in shared memory (n_eq is large here)."""
    net = ONE_PRODUCT[name]
    plan = nn_emul_plan(net.program(8))
    return max(o for o in range(2, 16) if nn_expected(plan, net.n_eq, o, OP_BATCH)["fits"])
OP_BATCH = 7  # odd: the last CTA owns lane 6 alone, its second owner thread is clamped to that lane


# ---- GPU: dense networks against the reference ---------------------------------------------------------------------

def _ki(ta):
    ki = ta._b.kernel_info()
    return {k: ki[k] for k in ("tape", "smem_bytes", "grid")}


@pytest.mark.gpu
@pytest.mark.parametrize("name,order", DENSE, ids=["%s@%d" % c for c in DENSE])
def test_dense_against_series_reference(name, order):
    """One step with write_tc: every Taylor coefficient within NN_BOUND of the 50-digit reference (normalised per
    variable and order), on the kernel setup_nn() must choose. Past the fit boundary the automatic selection takes a
    cooperative kernel, which meets the same bound, and asking for k_nn is refused."""
    net = CASES[name]
    st, ref = reference(name, order)
    P = net.program(order)
    e = nn_expected(nn_emul_plan(P), net.n_eq, order, REF_LANES)
    ta = hb.taylor_adaptive_batch(net.sys(), st, REF_LANES, tol=sr.order_tol(order))
    if e["fits"]:
        assert _ki(ta) == {k: e[k] for k in ("tape", "smem_bytes", "grid")}
    else:
        assert ta._b.kernel_info()["tape"] in ("smem", "global", "global-cta"), ta._b.kernel_info()
        with pytest.raises(ValueError, match="The dense-network kernel cannot run this program: it does not fit in "
                                             "shared memory"):
            ta._b.set_kernel("nn")
    ta.step(write_tc=True)
    err = sr.normalised_err(ta.tc, ref)
    print("%s@%d %s: normalised error %.3g" % (name, order, ta._b.kernel_info()["tape"], err))
    assert err < NN_BOUND, (name, order, err)


@pytest.mark.gpu
@pytest.mark.parametrize("idx", range(len(REFUSALS)), ids=REFUSALS)
def test_refusals_carry_the_planners_reason(idx):
    name, sys_, why = refusals()[idx]
    P = hb.Program(sys_, tol=sr.order_tol(8))
    plan = nn_emul_plan(P)
    st = np.random.default_rng(0).uniform(-1., 1., (P.n_eq, 3))
    ta = hb.taylor_adaptive_batch(sys_, st, 3, tol=sr.order_tol(8), pars=np.zeros((P.n_pars, 3)) if P.n_pars else None)
    assert ta._b.kernel_info()["tape"] != "nn"
    with pytest.raises(ValueError, match=re.escape("The dense-network kernel cannot run this program: " + plan["why"])):
        ta._b.set_kernel("nn")


@pytest.mark.gpu
def test_env_switch_keeps_automatic_selection_off_nn(monkeypatch):
    """HEYOKA_B200_NN=0, set before the batch is built: the automatic selection never takes k_nn; asking for it still
    works."""
    net = CASES["3:[13]"]
    st = net.states(5)
    monkeypatch.setenv("HEYOKA_B200_NN", "0")
    ta = hb.taylor_adaptive_batch(net.sys(), st, 5, tol=sr.order_tol(15))
    assert ta._b.kernel_info()["tape"] != "nn"
    ta._b.set_kernel("nn")
    assert ta._b.kernel_info()["tape"] == "nn"
    monkeypatch.delenv("HEYOKA_B200_NN")
    ta = hb.taylor_adaptive_batch(net.sys(), st, 5, tol=sr.order_tol(15))
    assert ta._b.kernel_info()["tape"] == "nn"


PROP_CASES = [n for n in CASES]
PROP_BATCH = 9


@pytest.mark.gpu
@pytest.mark.parametrize("name", PROP_CASES)
def test_propagate_until_against_oracle(name):
    """propagate_until() to per-lane final times (2-6 first steps) at order 15, on k_nn and on global-cta, against the
    oracle's FMA mode: identical step counts and outcomes, states to 1e-12."""
    net = CASES[name]
    P = net.program(15)
    st = net.states(PROP_BATCH, seed=3)
    o = oracle.OracleIntegrator(P, st, PROP_BATCH, mode=oracle.FMA)
    o.step()
    tf = np.linspace(2., 6., PROP_BATCH) * np.abs(o.last_h)
    o = oracle.OracleIntegrator(P, st, PROP_BATCH, mode=oracle.FMA)
    o.propagate_until(tf)
    for tape in ("nn", "global-cta"):
        ta = hb.taylor_adaptive_batch(net.sys(), st, PROP_BATCH, tol=sr.order_tol(15), kernel=dict(tape=tape))
        assert ta._b.kernel_info()["tape"] == tape
        ta.propagate_until(tf)
        assert [r[3] for r in ta.propagate_res] == [int(x) for x in o.n_steps], tape
        assert [r[0] for r in ta.propagate_res] == [int(x) for x in o.prop_outcome], tape
        assert np.array_equal(ta.time, o.t_hi), tape
        assert lane_err(ta.state, o.state) < 1e-12, tape


# ---- GPU: one-product networks, bit for bit against k_hbm ----------------------------------------------------------

def _snap(ta, tc=True):
    return dict(state=ta.state.copy(), t_hi=ta.dtime[0].copy(), t_lo=ta.dtime[1].copy(), last_h=ta.last_h.copy(),
                tc=ta.tc.copy() if tc and ta.tc is not None else None)


def _reset(ta, st):
    ta.state[:] = st
    ta.set_time(0.)


def _one_product_run(net, order, st, tape, lim_f, lim_b, tf, mdt, grid):
    """Every propagation path of a batch on kernel `tape`: results as plain arrays."""
    batch = st.shape[1]
    mk = lambda s=st: hb.taylor_adaptive_batch(net.sys(), s, batch, tol=sr.order_tol(order),  # noqa: E731
                                               kernel=dict(tape=tape))
    ta = mk()
    assert ta._b.kernel_info()["tape"] == tape
    out = {}
    ta.step(write_tc=True)
    out["step"] = _snap(ta) | {"res": list(ta.step_res)}
    for key, lim in (("fwd", lim_f), ("bwd", lim_b)):
        _reset(ta, st)
        ta.step(lim, write_tc=True)
        out[key] = _snap(ta) | {"res": list(ta.step_res)}
    _reset(ta, st)
    ta.propagate_until(tf, write_tc=True)
    out["prop"] = _snap(ta) | {"res": list(ta.propagate_res)}
    _reset(ta, st)
    ta.propagate_until(tf, max_delta_t=mdt)
    out["prop_mdt"] = _snap(ta, tc=False) | {"res": list(ta.propagate_res)}
    _reset(ta, st)
    ta.propagate_until(10. * tf, max_steps=7)
    out["max_steps"] = _snap(ta, tc=False) | {"res": list(ta.propagate_res)}
    for key, kw in (("grid_mdt", dict(max_delta_t=mdt)), ("grid_steps", dict(max_steps=3)), ("grid", dict())):
        g = mk()
        out[key] = dict(ret=g.propagate_grid(grid, **kw)) | _snap(g, tc=False) | {"res": list(g.propagate_res)}
    c = mk()
    co = c.propagate_until(tf, c_output=True)
    times = co.get_times()
    out["cout"] = dict(times=times, tcs=co.get_tcs(), at_grid=np.array([co(grid[k]).copy() for k in range(len(grid))]),
                       at_steps=np.array([co(times[k]).copy() for k in range(len(times) - 1)]))
    return out


def _same(a, b):
    if isinstance(a, np.ndarray):
        return np.array_equal(a, b, equal_nan=True)
    return a == b


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(ONE_PRODUCT))
def test_one_product_bit_for_bit_against_hbm(name):
    """Every neuron has one product: the matrix product adds exact zeros to one rounded product, tanh, tanh^2, the
    division by n + 1, the step size and the update follow the generic kernels' arithmetic. So k_nn equals k_hbm bit for
    bit on a free step, clamped steps, propagate_until() (write_tc, max_delta_t, max_steps), propagate_grid() and
    continuous output."""
    net, order = ONE_PRODUCT[name], op_order(name)
    P = net.program(order)
    st = net.states(OP_BATCH, seed=4)
    o = oracle.OracleIntegrator(P, st, OP_BATCH, mode=oracle.FMA)
    o.step()
    h = np.abs(o.last_h)
    tf = np.linspace(2., 6., OP_BATCH) * h
    grid = np.linspace(0., 6., 13)[:, None] * h[None, :]
    ref = _one_product_run(net, order, st, "hbm", 0.5 * h, -0.5 * h, tf, 0.4 * h, grid)
    got = _one_product_run(net, order, st, "nn", 0.5 * h, -0.5 * h, tf, 0.4 * h, grid)
    for phase, r in ref.items():
        for k, v in r.items():
            if v is not None:
                assert _same(got[phase][k], v), (phase, k)


def _one_product_source(net, s):
    """The input that state variable s of a one-product network reads, through one neuron per layer."""
    idx = net.outs[s]
    for W, _ in reversed(net.wb):
        idx = int(np.flatnonzero(W[idx])[0])
    return idx


@pytest.mark.gpu
def test_one_product_nan_lane_in_last_cta():
    """A NaN state in lane n - 1 of an odd batch: the last CTA owns that lane alone, and its second owner thread is
    clamped to the same lane with valid = false. The NaN goes in each state variable in turn. step() and
    propagate_until() fail that lane only, with k_hbm's outcome and step count; the other lanes keep the bits of k_hbm.

    The NaN lane itself follows the divergence stated in the header of nn_kernel.cuh. In k_hbm the NaN reaches only the
    state variables whose jet reads it (x_j itself and, order by order, the state variables fed by those), and the step
    size is NaN only if state variable 0 is one of them: the norms start from state variable 0, and std_max() keeps a NaN in its first argument
    and drops one in its second. In k_nn the matrix product multiplies the zero weights too (0 NaN = NaN), so every
    state variable of the lane, its step size and its time become NaN. Where state variable 0 reads the NaN, the two
    kernels agree bit for bit."""
    name = "op 13:[13]"
    net = ONE_PRODUCT[name]
    order = op_order(name)
    base = net.states(OP_BATCH, seed=5)
    bad = OP_BATCH - 1
    ok = np.arange(OP_BATCH) != bad
    src = np.array([_one_product_source(net, s) for s in range(net.n_eq)])
    seen = set()
    for j in range(net.n_eq):
        st = base.copy()
        st[j, bad] = np.nan
        # The state variables whose jet reads x_j: x_s^[k] reads x_src(s)^[0..k-1], so x_s's coefficients up to the
        # order read x_j iff j = src^k(s) for some k <= order.
        reads, cur = np.zeros(net.n_eq, dtype=bool), np.arange(net.n_eq)
        for _ in range(order + 1):
            reads |= cur == j
            cur = src[cur]
        res = {}
        for tape in ("hbm", "nn"):
            # (The constructor refuses a non-finite state: the NaN goes into the state mirror, uploaded at every call.)
            ta = hb.taylor_adaptive_batch(net.sys(), np.nan_to_num(st), OP_BATCH, tol=sr.order_tol(order),
                                          kernel=dict(tape=tape))
            ta.state[:] = st
            ta.step(write_tc=True)
            r = dict(step=_snap(ta) | {"res": [x[0] for x in ta.step_res]})
            _reset(ta, st)
            ta.propagate_until(np.full(OP_BATCH, 1.))
            r["prop"] = _snap(ta, tc=False) | {"res": [x[0] for x in ta.propagate_res],
                                               "n": [x[3] for x in ta.propagate_res]}
            res[tape] = r
        assert res["nn"]["prop"]["n"] == res["hbm"]["prop"]["n"], j
        for phase in ("step", "prop"):
            a, b = res["nn"][phase], res["hbm"][phase]
            assert a["res"] == b["res"] and a["res"][bad] == NF, (j, phase)
            for k in ("state", "t_hi", "t_lo", "last_h"):
                assert np.array_equal(a[k][..., ok], b[k][..., ok]), (j, phase, k)
            if a["tc"] is not None:
                assert np.array_equal(a["tc"][..., ok], b["tc"][..., ok]), (j, phase)
            # The NaN lane. k_nn: everything NaN.
            assert np.all(np.isnan(a["state"][:, bad])), (j, phase)
            assert np.isnan(a["last_h"][bad]) and np.isnan(a["t_hi"][bad]), (j, phase)
            if reads[0]:
                # k_hbm's step size is NaN as well: the same bits.
                for k in ("state", "t_hi", "last_h"):
                    assert _same(a[k][..., bad], b[k][..., bad]), (j, phase, k)
                seen.add("same")
            else:
                # k_hbm: a finite step, NaN exactly in the state variables that read x_j.
                assert np.isfinite(b["last_h"][bad]) and np.isfinite(b["t_hi"][bad]), (j, phase)
                assert np.array_equal(np.isnan(b["state"][:, bad]), reads), (j, phase, b["state"][:, bad])
                seen.add("diverges")
    assert seen == {"same", "diverges"}, seen


# ---- GPU: batch tails, persistence and sharding --------------------------------------------------------------------

TAIL_CASES = ["1:[3]", "5:[12,12]", "3:[130]", "4:[72]"]  # masked k, second chain, items > threads, 2 tiles per warp
N_BASE = 7


@pytest.mark.gpu
@pytest.mark.parametrize("name", TAIL_CASES)
def test_batch_tails_and_persistence(name):
    """Batch sizes 1, 2, 3, 265 (one CTA takes a second chunk) and 4 x 132 + 3 (every CTA at least two): every lane
    equals, bit for bit, the same lane run alone in a batch of 1, for a step with write_tc, a clamped step and
    propagate_until() (state, time, last_h, tc and results)."""
    net = CASES[name]
    order = 15
    P = net.program(order)
    base = net.states(N_BASE, seed=6)
    o = oracle.OracleIntegrator(P, base, N_BASE, mode=oracle.FMA)
    o.step()
    h = np.abs(o.last_h)
    tf_base, lim_base = np.linspace(3., 9., N_BASE) * h, -0.5 * h

    def run(idx):
        st = base[:, idx]
        batch = len(idx)
        ta = hb.taylor_adaptive_batch(net.sys(), st, batch, tol=sr.order_tol(order))
        e = nn_expected(nn_emul_plan(P), net.n_eq, order, batch)
        assert _ki(ta) == {k: e[k] for k in ("tape", "smem_bytes", "grid")}
        ta.step(write_tc=True)
        r = dict(step=_snap(ta) | {"res": list(ta.step_res)})
        _reset(ta, st)
        ta.step(lim_base[idx], write_tc=True)
        r["lim"] = _snap(ta) | {"res": list(ta.step_res)}
        _reset(ta, st)
        ta.propagate_until(tf_base[idx])
        r["prop"] = _snap(ta, tc=False) | {"res": list(ta.propagate_res)}
        return r

    alone = [run(np.array([i])) for i in range(N_BASE)]
    for batch in (1, 2, 3, 265, 4 * H100_SMS + 3):
        idx = np.arange(batch) % N_BASE
        r = run(idx)
        for phase in ("step", "lim", "prop"):
            for k in ("state", "t_hi", "t_lo", "tc", "last_h"):
                if alone[0][phase][k] is None or (phase == "prop" and k == "last_h"):
                    continue
                exp = np.stack([a[phase][k][..., 0] for a in alone], axis=-1)[..., idx]
                assert np.array_equal(r[phase][k], exp), (batch, phase, k, np.argwhere(r[phase][k] != exp)[:4])
            assert r[phase]["res"] == [alone[i][phase]["res"][0] for i in idx], (batch, phase)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["3:[130]", "3:[13]-shared"])
def test_sharded_equals_single_device(name):
    """A batch sharded in two on one device (device=[0, 0]) runs k_nn on both shards and equals the single-device
    batch bit for bit: a step with write_tc and propagate_until()."""
    net = CASES[name]
    batch = 11
    st = net.states(batch, seed=8)
    out = []
    for dev in (-1, [0, 0]):
        ta = hb.taylor_adaptive_batch(net.sys(), st, batch, tol=sr.order_tol(15), device=dev)
        assert ta._b.kernel_info()["tape"] == "nn" and ta._b.n_shards == (0 if dev == -1 else 2)
        ta.step(write_tc=True)
        s = _snap(ta) | {"res": list(ta.step_res)}
        ta.propagate_until(ta.time + 3. * np.abs(ta.last_h))
        out.append((s, _snap(ta, tc=False) | {"res": list(ta.propagate_res)}))
    for a, b in zip(*out):
        for k, v in a.items():
            if v is not None:
                assert _same(b[k], v), k
