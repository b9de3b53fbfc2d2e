"""Event detection on the device over the families of tests/event_root_cases.py: against the exact real roots of the
device's own event polynomials (tests/root_ref.py, the criteria of tests/test_event_roots_cpu.py), and against the
oracle step by step. The device and the oracle run the same algorithm with the same IEEE operations, so on a clamped
step (h = max_delta_t, no pow()) every output must be the oracle's bits: the records, the order, the state, the time
(hi, lo), last_h, the outcomes, the cooldown arrays and the Taylor coefficients. On free steps h is held to 4 ulps and the
rest to the tolerances of tests/test_gpu_events.py."""
import numpy as np
import pytest

import event_root_cases as erc
import heyoka_b200 as hb
import oracle
from test_event_roots_cpu import KNOWN_FINDINGS

pytestmark = pytest.mark.gpu
FAMILIES = erc.families()


def dev(*a, **k):
    return hb.taylor_adaptive_batch(*a, **k)


def orc(*a, **k):
    return oracle.OracleEventIntegrator(*a, **k)


def _bits(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).view(np.int64)


def _recs(ta):
    return [(e[0], e[1], e[2], e[3], float(e[4]).hex(), float(e[5]).hex()) for e in ta._b.events()]


def snapshot(fam, ta):
    """Every output of an event step, floats as bit patterns."""
    out = {"events": _recs(ta), "order": ta.get_order(), "state": _bits(ta.state), "t_hi": _bits(ta.dtime[0]),
           "t_lo": _bits(ta.dtime[1]), "last_h": _bits(ta.last_h), "outcome": [r[0] for r in ta.step_res],
           "tc_events": _bits(ta._b.tc_events(fam.n_ev)), "tc": _bits(ta._b.tc())}
    if fam.n_te:
        a, s, c = ta._b.cooldowns(fam.n_te)
        out.update(cd_on=np.asarray(a, dtype=np.int64), cd_spent=_bits(s), cd_val=_bits(c))
    return out


def trace(fam, mk, lanes=None):
    snaps = []
    erc.run(fam, mk, lanes=lanes, on_step=lambda k, ta, cd, m: snaps.append(snapshot(fam, ta)))
    return snaps


def assert_same_bits(fam, a, b, what):
    for k, (x, y) in enumerate(zip(a, b)):
        for key in x:
            xv, yv = x[key], y[key]
            same = np.array_equal(xv, yv) if isinstance(xv, np.ndarray) else xv == yv
            assert same, "%s: %s, step %d: %s differs" % (fam.name, what, k, key)


def assert_close(fam, g, o):
    """Free steps: h to 4 ulps, the rest to the tolerances of tests/test_gpu_events.py."""
    for k, (x, y) in enumerate(zip(g, o)):
        hg, ho = x["last_h"].view(np.float64), y["last_h"].view(np.float64)
        assert np.all(np.abs(hg - ho) <= 4 * np.spacing(np.abs(ho))), (fam.name, k, hg, ho)
        assert [e[:4] for e in x["events"]] == [e[:4] for e in y["events"]], (fam.name, k)
        for a, b in zip(x["events"], y["events"]):
            assert abs(float.fromhex(a[4]) - float.fromhex(b[4])) <= 2e-12 * abs(ho[a[0]]) + 1e-15, (fam.name, k)
        assert x["outcome"] == y["outcome"], (fam.name, k)
        assert np.max(np.abs(x["state"].view(np.float64) - y["state"].view(np.float64))) < 1e-12
        pw = np.arange(fam.order + 1)[None, :, None]
        hh = np.minimum(np.maximum(np.abs(ho), 1e-300)[None, None, :] ** pw, 1.0)
        d = np.abs(x["tc_events"].view(np.float64) - y["tc_events"].view(np.float64)).reshape(fam.n_ev, fam.order + 1, -1)
        assert np.max(d * hh) < 1e-12, (fam.name, k)


@pytest.mark.parametrize("fam", FAMILIES, ids=lambda f: f.name)
def test_device_against_oracle(fam):
    g, o = trace(fam, dev), trace(fam, orc)
    assert len(g) == len(o) == len(fam.mdts)
    if fam.clamped:
        assert_same_bits(fam, g, o, "device vs oracle")
    else:
        assert_close(fam, g, o)


@pytest.mark.parametrize("fam", FAMILIES, ids=lambda f: f.name)
def test_device_against_exact_roots(fam):
    problems, findings, n_well = [], [], 0
    lanes = erc.sample_lanes(fam.B)

    def on_step(k, ta, cd, m):
        nonlocal n_well
        p, n, f, w = erc.against_exact_roots(fam, ta, cd, lanes)
        problems.extend(p)
        findings.extend(f)
        n_well += w

    erc.run(fam, dev, on_step=on_step)
    assert not problems, "\n".join(problems)
    assert n_well >= 1
    assert len(findings) == KNOWN_FINDINGS.get(fam.name, 0), findings


def _simple_k5(B):
    rng = np.random.default_rng(B)
    return erc.Family("simple_K5_B%d" % B, 33, rng.uniform(-0.1, 0.1, B), erc._sorted_roots(rng, 5, B, 0.03, 1.97, 0.02),
                      ntes=[(erc._product_event(5), erc.ANY)], tes=[(erc._product_event(2), 0.1, erc.POS)],
                      mdts=(1.0, 1.0, 1.0))


@pytest.mark.parametrize("B", [1, 5, 31, 33, 257])
def test_batch_sizes(B):
    """Bit for bit against the oracle (whose lanes are independent by construction) at batch sizes around the warp and
    block boundaries; every lane (up to 33 lanes; lanes at warp boundaries of the 257-lane batch) also gives the bits of
    the same lane run alone on the device."""
    fam = _simple_k5(B)
    g = trace(fam, dev)
    assert_same_bits(fam, g, trace(fam, orc), "device vs oracle")
    assert_lanes_alone(fam, g, range(B) if B <= 33 else [0, 1, 31, 32, 63, 64, 128, 255, 256])


def assert_lanes_alone(fam, g, lanes):
    """Each of the given lanes of the batch trace g gives the bits of the same lane run alone on the device."""
    B = fam.B
    for lane in lanes:
        alone = trace(fam, dev, lanes=[lane])
        for k in range(len(g)):
            assert [e[1:] for e in g[k]["events"] if e[0] == lane] == [e[1:] for e in alone[k]["events"]], (lane, k)
            for key in ("state", "t_hi", "t_lo", "last_h", "tc_events"):
                assert np.array_equal(g[k][key].reshape(-1, B)[:, lane], alone[k][key].reshape(-1)), (lane, k, key)


def test_record_overflow():
    """64 lanes x 20 roots = 1280 records against a record array of 1024: the step grows the array and redoes the
    detection. Bit for bit against the oracle and against the same lanes run 16 at a time (no overflow)."""
    fam = erc.overflow_family()
    g = trace(fam, dev)
    assert len(g[0]["events"]) > max(fam.B * fam.n_ev, 1024)
    assert_same_bits(fam, g, trace(fam, orc), "device vs oracle")
    for b0 in range(0, fam.B, 16):
        part = trace(fam, dev, lanes=list(range(b0, b0 + 16)))
        exp = [(e[0] - b0,) + e[1:] for e in g[0]["events"] if b0 <= e[0] < b0 + 16]
        assert part[0]["events"] == exp
        assert np.array_equal(part[0]["tc_events"].reshape(-1, 16), g[0]["tc_events"].reshape(-1, fam.B)[:, b0:b0 + 16])


def test_many_candidates():
    """8500 (event, lane) candidates, more than the 64 x 132 detection threads: threads loop over candidates."""
    fam = erc.many_candidates_family()
    g = trace(fam, dev)
    assert_same_bits(fam, g, trace(fam, orc), "device vs oracle")
    # Lanes on both sides of the 8448 candidates the first pass of the detection threads covers.
    assert_lanes_alone(fam, g, [0, 1, 4000, 8447, 8448, 8449, 8499])


def test_order_48_refused():
    """The same error class on one device and on a batch made of two shards."""
    x, = hb.make_vars("x")
    for kw in ({}, {"device": [0, 0]}):
        hb.taylor_adaptive_batch([(x, hb.expression(1.0))], np.zeros((1, 2)), 2, tol=5e-40,
                                 nt_events=[hb.nt_event_batch(x - 0.5, lambda ta, t, d, i: None)], **kw)
        with pytest.raises(NotImplementedError, match="Event detection supports Taylor orders up to 47"):
            hb.taylor_adaptive_batch([(x, hb.expression(1.0))], np.zeros((1, 2)), 2, tol=1e-40,
                                     nt_events=[hb.nt_event_batch(x - 0.5, lambda ta, t, d, i: None)], **kw)
