"""CPU: the exact references of tests/test_vector_cones_exact_gpu.py (tests/vector_exact.py) are the projections they
claim to be, and their gate rejects the defects the second-order, box and l1 kernels could have.

* every reference meets Moreau's conditions exactly: Pi in K, Pi - v in the polar cone (up to sign and metric) and
  <Pi, Pi - v> = 0, the box's in its metric diag(rho);
* the box's exact Newton (the reference's iteration and stop rules) reaches the sorted-breakpoint root, within 20 of
  its 25 steps from the warm start each call sees;
* the l1 threshold's integer path is the Fraction path, Michelot's last pass is the sorted scan's threshold, and both
  agree with tests/spectral_numpy.py;
* five planted defects, applied to the exact answers, exceed the gate by at least 100x: a big SOC cone that drops its
  last chunk's partial sum, a head written from the unscaled value, a cone-per-item cap off by one, an l1 threshold
  one Michelot pass early and a box applied with the t of one Newton step earlier."""
from fractions import Fraction

import numpy as np
import pytest

import eigen_exact as ee
import spectral_numpy
import vector_exact as ve
from scs_b200 import problems


@pytest.mark.parametrize("q", [q for q in ve.SOC_SIZES if q <= 12289])
def test_soc_references_are_the_projections(q):
    kinds = set()
    for name, b in ve.soc_size_blocks(q):
        assert ve.moreau_soc(b), (q, name)
        if q >= 2:
            s, v1 = b.parts["s"], int(b.v[0])
            kinds.add("in" if s <= v1 else ("polar" if s <= -v1 else "between"))
            assert s * s == int((b.v[1:].astype(object) ** 2).sum())
        if b.N:  # the float restatement of scs_b200/problems.py agrees
            num = problems.proj_cone(b.v.astype(np.float64), {"q": [b.N]}) - b.v
            assert np.abs(num - b.out).max() <= 1e-12 * max(1.0, float(np.abs(b.v).max())), (q, name)
    if q >= 3:
        assert kinds == {"in", "polar", "between"}


@pytest.mark.parametrize("n", [1, 255, 256, 257, 8191, 8193])
def test_ell1_references_are_the_projections(n):
    passes = 0
    for name, b in ve.ell1_size_blocks(n):
        assert ve.moreau_ell1(b), (n, name)
        T, mu, mus = b.parts["T"], b.parts["mu"], b.parts["mus"]
        a = np.abs(b.v[1:])
        if n <= 257:  # the integer path is the Fraction path
            assert ee.ell1_threshold(Fraction(T), [Fraction(int(x)) for x in a]) == mu, (n, name)
        # Michelot's iteration ends on the sorted scan's threshold
        assert (mus is None) == (mu is None) and (mus == [] if mu == 0 else mus is None or mus[-1] == mu), (n, name)
        passes = max(passes, len(mus or []))
        tn, pn = spectral_numpy.proj_ell1(float(T), b.v[1:].astype(np.float64))
        pi = b.out + b.v
        assert abs(tn - pi[0]) <= 1e-12 * max(1.0, abs(tn)), (n, name)
        assert np.abs(pn - pi[1:]).max(initial=0) <= 1e-12 * max(1.0, float(a.max(initial=0))), (n, name)
    if n >= 255:
        assert passes >= 3, passes
        tie = dict(ve.ell1_size_blocks(n))["tie"]
        assert (np.abs(tie.v[1:]) == tie.parts["mu"]).sum() >= 1


def _box_cases():
    return [(name, w) for name in ("plain", "inf", "inf_D", "zero", "far") for w in (False, True)]


@pytest.mark.parametrize("name,weighted", _box_cases())
@pytest.mark.parametrize("n", [1, 2, 300])
def test_box_references_are_the_projections(name, weighted, n):
    b = ve.box_case(name, n, weighted)
    bp, t = b.parts["bp"], b.parts["t"]
    assert ve.moreau_box(b), (name, weighted, n)
    assert bp.root() == t
    its = b.parts["its"]
    assert its.index(t) + 1 <= ve.NEWTON_STEPS_ALLOWED and len(its) <= ve.BOX_MAX_ITERS
    if name == "zero":
        assert t == 0
    if name in ("inf", "inf_D") and n >= 300:
        assert (~bp.lfin).any() and (~bp.ufin).any()
    if name == "inf_D":
        bl, bu, D = ve.box_library_bounds(b)
        # the library's scaling (host/cone_setup.c b200_normalize_box) turns the given bounds into those of the block
        f = D[1:] / D[0]
        for j in range(n):
            assert (bu[j] >= 1e15 and bp.bu[j] == ve.INF) or Fraction(bu[j]) * Fraction(f[j]) == bp.bu[j]
            assert (bl[j] <= -1e15 and bp.bl[j] == -ve.INF) or Fraction(bl[j]) * Fraction(f[j]) == bp.bl[j]


def test_box_warm_sequence_and_bounds_equal():
    seq = ve.box_warm_sequence()
    ts = [b.parts["t"] for b in seq]
    assert ts[1] == ts[0] * 2 ** 40 and ts[2] == ts[0]
    for b in seq:
        assert ve.moreau_box(b)
        assert b.parts["bp"].root() == b.parts["t"]
    bp = seq[0].parts["bp"]
    assert any(l == u for l, u in zip(bp.bl, bp.bu))


# ---------------------------------------------------------------------------------------------- planted defects
def _soc_dropped_last_chunk(b):
    """the big cone's norm without its last 4096-row chunk's partial"""
    v1, tail = int(b.v[0]), b.v[1:].astype(np.float64)
    last = ((b.N - 1) // ve.SOC_CHUNK) * ve.SOC_CHUNK   # first row of the last chunk
    s = float(np.sqrt((tail[:last - 1] ** 2).sum()))
    a = (s + v1) / 2
    return np.concatenate(([a - v1], (a / s - 1) * tail)) if -s < v1 < s else None


def test_gate_rejects_planted_defects():
    ratios = {}
    # SOC: a big cone (33 chunks, the last of one row) drops its last chunk's partial
    for name, b in ve.soc_size_blocks(131073):
        if name == "mid":
            d = _soc_dropped_last_chunk(b)
            assert b.ratio(b.ref()) <= 0.05
            ratios["soc last chunk dropped"] = b.ratio(d)
            # the head written from the unscaled value: Pi_0 = v_1, so Pi_0 - v_1 = 0
            d = b.out.copy()
            d[0] = 0.0
            ratios["soc head unscaled"] = b.ratio(d)
    # cone-per-item cap off by one: 4097 rays, the cone after the cap left as it came in (-r x = v)
    rng = np.random.default_rng(5)
    rays = [ve.soc_block(1, "below_polar", rng) for _ in range(ve.SOC_ITEM_CONES + 1)]
    cap = rays[ve.SOC_ITEM_CONES]
    for r in (1.0, 4.0, 0.125):
        ratios[f"soc cone cap off by one, r={r}"] = cap.ratio(cap.v.astype(np.float64), r)
    # l1: the threshold of one Michelot pass earlier
    for n in (257, 8193, 131073):
        b = dict(ve.ell1_size_blocks(n))["between"]
        mus = b.parts["mus"]
        assert len(mus) >= 2
        d = ve.ell1_out(b.parts["T"], b.v[1:], mus[-2])
        assert b.ratio(b.ref()) <= 0.05
        ratios[f"l1 one pass early, n={n}"] = b.ratio(d)
    # box: the t of one Newton step earlier
    for name in ("plain", "inf_D", "far"):
        b = ve.box_case(name, 300)
        its = b.parts["its"]
        k = its.index(b.parts["t"])
        assert k >= 1
        assert b.ratio(b.ref()) <= 0.05
        ratios[f"box one Newton step early, {name}"] = b.ratio(b.parts["bp"].out(its[k - 1]))
    print({k: f"{v:.3g}" for k, v in ratios.items()})
    bad = {k: v for k, v in ratios.items() if not v >= 100}
    assert not bad, bad
