"""Event detection of the CPU oracle against the exact real roots of the event polynomials (tests/root_ref.py), over the
families of tests/event_root_cases.py. No GPU needed.

Completeness: every well-conditioned root in the step (its tolerance, derived from the Horner error bound, at least
root_ref.WELL_MARGIN = 16 times smaller than its distance to every other root, complex ones included, to the ends of
the step and to a cooldown boundary) that passes the direction and cooldown filters gives exactly one record, with the
right derivative sign, within the tolerance. No spurious events: every record lies within the tolerance of a real root.
The roots the check does not apply to (clusters, even multiplicities, step ends, complex pairs next to the real axis) are
named with what the oracle does there (pytest -s prints them). Known departures of the shared algorithm from the exact
answer are pinned, not skipped: see KNOWN_FINDINGS."""
import numpy as np
import pytest

import event_root_cases as erc
import heyoka_b200 as hb
import oracle
import root_ref

FAMILIES = erc.families()


def make(*a, **k):
    return oracle.OracleEventIntegrator(*a, **k)


# Families where the shared algorithm departs from the exact answer, with how many such findings the oracle run gives.
# A root exactly on a point the bisection reaches (the start of the step, or tau = 1/2) is reported more than once, and
# the next root of the isolating interval that begins at a root at t = 0 is not reported (root_ref.check()).
KNOWN_FINDINGS = {"root_at_start": 2, "chebyshev_T5": 1}


def run_family(fam, lanes=None):
    res = {"problems": [], "notes": [], "findings": [], "n_well": 0, "n_rec": [], "starts": 0, "clamps": 0,
           "cuts": 0, "backward": False}
    lanes = erc.sample_lanes(fam.B) if lanes is None else lanes
    oracle.ev_max_depth()

    def on_step(k, ta, cd, mdt):
        evs = ta._b.events()
        res["n_rec"].append(len(evs))
        res["starts"] += sum(e[4] == 0.0 for e in evs)
        if mdt is not None:
            # A clamped record: at nextafter(h, 0) while the exact root rounds to h itself, so fl(tau h) was h (a
            # genuine root at nextafter(h, 0), as in root_at_end, does not count).
            tce = ta._b.tc_events(fam.n_ev)
            for e in evs:
                h = mdt[e[0]]
                if e[4] == np.nextafter(h, 0.0):
                    k = e[1] if e[2] else fam.n_te + e[1]
                    rs = root_ref.exact_roots(tce[k, :, e[0]], h)
                    res["clamps"] += int(any(R.in_step and float(R.t) == h for R in rs))
            res["backward"] |= bool(np.any(mdt < 0) and len(evs) > 0)
        if cd is not None:
            a, s, c = cd
            for k2 in range(fam.n_te):
                for lane in range(fam.B):
                    if a[k2, lane] and mdt is not None:
                        cut = root_ref.cooldown_cut(mdt[lane], 1, s[k2, lane], c[k2, lane])
                        res["cuts"] += int(0 < cut < abs(mdt[lane]) and abs(ta.last_h[lane]) > cut)
        p, n, f, w = erc.against_exact_roots(fam, ta, cd, lanes)
        res["problems"] += p
        res["notes"] += n
        res["findings"] += f
        res["n_well"] += w

    ta = erc.run(fam, make, on_step=on_step)
    res["depth"] = oracle.ev_max_depth()
    res["order"] = ta.get_order()
    return res


_RESULTS = {}


def results(fam):
    if fam.name not in _RESULTS:
        _RESULTS[fam.name] = run_family(fam)
    return _RESULTS[fam.name]


@pytest.mark.parametrize("fam", FAMILIES, ids=lambda f: f.name)
def test_oracle_against_exact_roots(fam):
    r = results(fam)
    for s in r["notes"]:
        print("  ", s)
    assert not r["problems"], "\n".join(r["problems"])
    assert r["n_well"] >= 1, "%s: no root the completeness check applies to (a bad family)" % fam.name
    assert len(r["findings"]) == KNOWN_FINDINGS.get(fam.name, 0), r["findings"]


@pytest.mark.parametrize("fam", FAMILIES, ids=lambda f: f.name)
def test_isolation_depth_below_device_stack(fam):
    """The device keeps the isolation's working list in a stack of EV_STACK = 48 entries and drops the (event, lane)
    that would overflow it; the oracle's list never gets near that on these families (close pairs down to 2^-52,
    double and triple roots, orders 3 to 47)."""
    assert results(fam)["depth"] < 48, (fam.name, results(fam)["depth"])


def test_clamped_families_are_clamped():
    """The families marked clamped have event polynomials of degree below p - 1, so orders p and p - 1 of every row
    are zero and the step size is max_delta_t exactly (no pow())."""
    for fam in FAMILIES:
        if not fam.clamped:
            continue
        ta = fam.build(make)
        ta.step(max_delta_ts=fam.mdt(0))
        p = ta.get_order()
        tce, tcs = ta._b.tc_events(fam.n_ev), ta._b.tc()
        assert np.all(tce[:, p - 1:, :] == 0) and np.all(tcs[:, p - 1:, :] == 0), fam.name


def test_large_families_against_exact_roots():
    """The record-overflow family (64 lanes x 20 roots) and the many-candidates family (8500 lanes), lanes sampled."""
    for fam in (erc.overflow_family(), erc.many_candidates_family()):
        r = run_family(fam, lanes=erc.sample_lanes(fam.B, 3))
        assert not r["problems"], "\n".join(r["problems"])
        assert r["n_well"] >= 1 and r["depth"] < 48
        _RESULTS[fam.name] = r


def test_paths_reached():
    """The families reach every path of the device's event step that used to go untested (checked on the oracle's
    results): more records in one step than the device's record array (max(B n_ev, 1024)); more candidates than
    64 x 132 detection threads; a root at the start of a step; a root clamped to h (a subnormal step: see
    root_clamped_to_h); a cooldown boundary inside a step; a backward step; orders 3 and 47."""
    for fam in (erc.overflow_family(), erc.many_candidates_family()):
        if fam.name not in _RESULTS:
            _RESULTS[fam.name] = run_family(fam, lanes=[0])
    ov, mc = erc.overflow_family(), erc.many_candidates_family()
    assert max(_RESULTS[ov.name]["n_rec"]) > max(ov.B * ov.n_ev, 1024)
    # Every lane has its root in the step: every (event, lane) pair is a candidate.
    assert _RESULTS[mc.name]["n_rec"][0] == mc.B > 64 * 132
    rs = [results(f) for f in FAMILIES]
    assert sum(r["starts"] for r in rs) > 0
    assert sum(r["clamps"] for r in rs) > 0
    assert sum(r["cuts"] for r in rs) > 0
    assert any(r["backward"] for r in rs)
    assert {3, 47} <= {r["order"] for r in rs}


def test_checker_catches_direction_and_cooldown_slips():
    """root_ref.check() on synthetic records for t^2 - t + 0.21 over h = 1 (crossings: -1 at 0.3, +1 at 0.7): the
    right records pass; a record against the requested direction, a record in the cooldown, a missing record, a
    duplicate, a wrong derivative sign and a record away from every root all fail."""
    roots = root_ref.exact_roots([0.21, -1.0, 1.0], 1.0)
    a, b = [R.tf for R in roots if R.in_step]
    assert abs(a - 0.3) < 1e-15 and abs(b - 0.7) < 1e-15 and [R.sgn for R in roots if R.in_step] == [-1, 1]

    def n_problems(records, direction=0, cut=0.0):
        return len(root_ref.check(records, roots, 1.0, direction, cut)[0])

    both = [(a, -1), (b, 1)]
    assert n_problems(both) == 0
    assert n_problems([(b, 1)], direction=1) == 0
    assert n_problems([(a, -1)], direction=-1) == 0
    assert n_problems([(b, 1)], cut=0.5) == 0
    assert n_problems(both, direction=1) > 0        # a is crossed downwards
    assert n_problems(both, direction=-1) > 0       # b is crossed upwards
    assert n_problems(both, cut=0.5) > 0            # a is in the cooldown
    assert n_problems([(a, -1)]) > 0                # b missing
    assert n_problems(both + [(b, 1)]) > 0          # b twice
    assert n_problems([(a, 1), (b, 1)]) > 0         # wrong sign at a
    assert n_problems(both + [(0.5, 1)]) > 0        # no root at 0.5
    assert n_problems([(a + 1e-9, -1), (b, 1)]) > 0  # beyond the tolerance of a


def test_order_47_is_the_limit():
    """tol = 5e-40 gives order 47, the highest order event detection supports (EV_MAXP1 = 48); 1e-40 gives 48, which
    the device refuses (tests/test_gpu_event_roots.py)."""
    assert hb.order_from_tol(5e-40) == 47 and hb.order_from_tol(1e-40) == 48
