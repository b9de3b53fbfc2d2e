"""CPU-side tests: the C ABI loads and exports every declared symbol, the symbolic front end and the
decomposition reproduce the reference's shapes, argument validation. No CUDA calls."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import heyoka_b200 as hb
from heyoka_b200 import _capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "heyoka_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    names = set(re.findall(r"\b(hy_[a-z0-9_]+)\s*\(", hdr))
    assert len(names) >= 35
    lib = C.CDLL(_capi.LIB_PATH)
    for n in sorted(names):
        assert hasattr(lib, n), "symbol %s declared in include/heyoka_b200.h but not exported" % n
    assert set(_capi.SIGNATURES) == names
    assert b"heyoka_b200" in _capi.lib.hy_version()


def test_expression_folding_rules():
    """src/expression_ops.cpp:45-92, src/math/sum.cpp:548-601, src/math/prod.cpp:913-975, pow.cpp:1024-1062."""
    x, y = hb.make_vars("x", "y")
    assert repr(hb.expression(2.) + hb.expression(3.)) == "5"
    assert repr(x + 0.) == "x" and repr(0. + x) == "x"
    assert repr(x * 1.) == "x" and repr(x * 0.) == "0"
    assert repr(x - y) == "sum(x, prod(-1, y))"
    assert repr(x / y) == "prod(x, pow(y, -1))"
    assert repr(-x) == "prod(-1, x)"
    assert repr(x * 2.) == "prod(2, x)"          # numbers first
    assert repr(x + 2. + 3.) == "sum(5, x)" or repr(x + 2. + 3.) == "sum(3, sum(2, x))"
    assert repr(hb.sum([x, 1., y, 2.])) == "sum(3, x, y)"
    assert repr(hb.prod([x, 2., y, 3.])) == "prod(6, x, y)"
    assert repr(x ** 1.) == "x" and repr(x ** 0.) == "1"
    assert repr(hb.expression(2.) ** 3.) == "8"
    assert repr(hb.sqrt(x)) == "pow(x, 0.5)"
    assert repr(hb.sin(hb.expression(0.))) == "0"


def test_decompose_sizes_reference_cases():
    """test/taylor_decompose.cpp:38-66 (sizes) + model-level shapes (SURVEY.md section 8 table)."""
    x, y = hb.make_vars("x", "y")
    assert hb.Program([(x, x)]).dc_size == 2
    assert hb.Program([(y, x + y), (x, x - y)]).dc_size == 6
    P = hb.Program([(x, hb.make_vars("v")[0]), (hb.make_vars("v")[0], -9.8 * hb.sin(x))])
    assert P.dc_size == 7 and "cos(u_0)" in P.dc_str() and "deps: 3" in P.dc_str()
    P = hb.Program(hb.model.nbody(2, masses=[1., 0.]))
    assert (P.n_eq, P.n_uvars) == (12, 21)
    P = hb.Program(hb.model.nbody(6))
    assert P.n_eq == 36
    from common import sys_outer_ss
    P = hb.Program(sys_outer_ss(), high_accuracy=True)
    assert (P.n_eq, P.n_uvars, P.order, P.n_pars) == (36, 234, 20, 0)
    c = P.costs()
    assert c["b_min"] == 8 * (2 * 36 + 0 + 7) and c["b_tape"] == c["b_min"] + 16 * (234 * 20 + 36)


def test_decompose_transformations():
    x, y, z = hb.make_vars("x", "y", "z")
    # sum of squares -> sum_sq; pow(., -1) in a product -> div; a + (-1*b) -> sub; pow(x, par) -> exp(par*log(x))
    s = hb.Program([(x, x ** 2. + y ** 2.), (y, x / y), (z, hb.pow(z, hb.par[0]))]).dc_str()
    assert "sum_sq(u_0, u_1)" in s and "div(u_0, u_1)" in s and "log(u_2)" in s and "exp(" in s
    # sums are split in chunks of 8, products in binary
    terms = [hb.expression("v%d" % i) for i in range(20)]
    vs = terms
    sysl = [(vs[i], hb.sum(vs) if i == 0 else vs[i]) for i in range(20)]
    s = hb.Program(sysl).dc_str()
    n_sum = [len(m.split(",")) for m in re.findall(r"= sum\((.*?)\)", s)]
    assert sorted(n_sum) == [3, 4, 8, 8]
    s = hb.Program([(x, hb.prod([x, y, z, x])), (y, y), (z, z)]).dc_str()
    assert all(len(m.split(",")) == 2 for m in re.findall(r"= prod\((.*?)\)", s))
    # CSE: the same subexpression built twice appears once
    s = hb.Program([(x, hb.sin(x + y)), (y, hb.sin(x + y) * 2.)]).dc_str()
    assert s.count("sin(") == 1 and s.count("cos(") == 1


def test_order_from_tol():
    """include/heyoka/detail/taylor_common.hpp:165-191 (values quoted in SURVEY.md section 3.1)."""
    assert hb.order_from_tol(np.finfo(float).eps) == 20
    assert hb.order_from_tol(1e-12) == 15
    assert hb.order_from_tol(1e-9) == 12
    assert hb.order_from_tol(0.9) == 2
    x, = hb.make_vars("x")
    assert hb.Program([(x, x)], tol=1e-12).order == 15


def test_error_conventions():
    x, y = hb.make_vars("x", "y")
    with pytest.raises(ValueError, match="not a variable"):
        hb.Program([(x + y, x)])
    with pytest.raises(ValueError, match="appears twice"):
        hb.Program([(x, x), (x, x)])
    with pytest.raises(ValueError, match="right-hand side but not in the left-hand side"):
        hb.Program([(x, y)])
    with pytest.raises(ValueError, match="must be finite and positive"):
        hb.Program([(x, x)], tol=-1.)
    with pytest.raises(ValueError, match="at least 2 bodies"):
        hb.model.nbody(1)
    with pytest.raises(NotImplementedError):
        hb._func("erf", x)
    # raw programs are validated
    with pytest.raises(ValueError, match="before its definition"):
        hb.Program.from_arrays(1, 2, 0, 20, [[8, 5, 0, 0]], [], [], [1])
    with pytest.raises(NotImplementedError, match="Unknown opcode"):
        hb.Program.from_arrays(1, 2, 0, 20, [[999, 0, 0, 0]], [], [], [1])


def test_no_cpu_fallback_without_device():
    """Without a CUDA device the compute entry points fail loudly with HY_ERR_CUDA."""
    import subprocess
    import sys
    code = ("import heyoka_b200 as hb\n"
            "x, = hb.make_vars('x')\n"
            "try:\n"
            "    hb.Batch(hb.Program([(x, x)]), 4)\n"
            "    print('CREATED')\n"
            "except hb.HyError as e:\n"
            "    print('HYERROR', e.code, e)\n")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=ROOT)
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True).stdout
    assert "HYERROR -3" in out and "no CPU fallback" in out


def test_null_batch_handle_is_an_invalid_argument():
    """Every hy_batch_* function that takes a batch handle and returns a status code refuses a NULL handle with
    HY_ERR_INVALID_ARG, before it touches a device (run in a subprocess without a device, so that a crash is a failure
    rather than the end of the test run)."""
    import subprocess
    import sys
    hdr = open(os.path.join(ROOT, "include", "heyoka_b200.h")).read()
    names = sorted(set(re.findall(r"\bint\s+(hy_batch_[a-z0-9_]+)\s*\(\s*(?:const\s+)?hy_batch\s*\*", hdr)))
    assert len(names) >= 29
    code = ("import ctypes as C\n"
            "from heyoka_b200 import _capi\n"
            "ints = (C.c_int, C.c_uint32, C.c_int64, C.c_uint64)\n"
            "for name in %r:\n"
            "    args = [0. if t is C.c_double else 0 if t in ints else None for t in _capi.SIGNATURES[name][1]]\n"
            "    print(name, getattr(_capi.lib, name)(*args), flush=True)\n" % (names,))
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=ROOT)
    res = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True)
    got = dict(line.split() for line in res.stdout.splitlines())
    assert res.returncode == 0, (res.returncode, sorted(set(names) - set(got)), res.stderr[-2000:])
    assert got == {n: str(_capi.HY_ERR_INVALID_ARG) for n in names}


def test_model_builders_decomposition_pinned():
    """heyoka_b200/csrc/model.cpp was rewritten in round 2 (table-driven pair enumeration, layer builder over index
    ranges): the expression trees - hence the Taylor decompositions - must be exactly what they were (hashes of
    hy_program_dc_str() recorded before the rewrite). The decomposition itself is pinned against the reference's sizes
    in test_oracle_golden.py / tests/cpp/test_batch_api.cpp (36 + 198 + 36 entries for the 6-body system)."""
    import hashlib
    from common import FFNN_TOL, sys_ffnn, sys_nbody32, sys_outer_ss, sys_two_body

    def h(sys_, **kw):
        return hashlib.sha1(hb.Program(sys_, **kw).dc_str().encode()).hexdigest()[:12]

    assert h(sys_outer_ss(), high_accuracy=True) == "573f3f3148f6"
    assert h(sys_two_body()) == "33f528fabe8c"
    assert h(sys_nbody32()) == "7d05336c9bb4"
    assert h(sys_ffnn(), tol=FFNN_TOL) == "fe21beab5461"
    assert h(hb.model.nbody(4)) == "afa50942f190"
    assert h(hb.model.nbody(3, masses=[1., 0.5])) == "65c79fb1d72c"
