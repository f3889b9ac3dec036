"""CPU checks of the iir_order.cu model (tests/iir_order_ref.py): the model of the kernel's decomposition stays within the
per-output bound for every filter of the GPU set, and each deliberate mutant breaks it by a clear margin."""
import numpy as np
import pytest

from oracle import lr_oracle as O
from tests import iir_order_ref as R

FILTERS = R.filters()
MUTANTS = ("power", "lookback", "xhist", "ystate32", "a0", "hom")
# ragged calls over several tiles, a call shorter than the longest filter, 0- and 1-sample calls
CALLS = (3 * R.T + 17, 0, 1, 40, R.T - 1, 5 * R.T + 3, 8192)


def _stream(cplx, seed=1):
    rng = np.random.default_rng(seed)
    xs = []
    for n in CALLS:
        v = rng.uniform(-1, 1, n)
        if cplx:
            v = v + 1j * rng.uniform(-1, 1, n)
        xs.append(v.astype(np.complex64 if cplx else np.float32))
    return xs


def _run(b, a, cplx, mutant=None):
    xs = _stream(cplx)
    _, ref, bnd = R.bound(b, a, xs, cplx)
    m = R.OrderModel(b, a, cplx, mutant)
    got = np.concatenate([m.process(x) for x in xs])
    return R.excess(got, ref, bnd)


def test_filter_set_shapes():
    for name, (b, a) in FILTERS.items():
        assert 1 <= len(b) <= 64 and 1 <= len(a) <= 64, name
        assert len(b) > 10 or len(a) > 10, name
        assert a[0] == 2.0, name


def test_reference_matches_oracle_recurrence():
    b, a = FILTERS["ellip5_bandpass"]
    x = _stream(False)[0][:3000]
    ref = R.reference(b, a, [x])
    orc = O.IIRFilter(b, a, False).process(x)
    assert np.max(np.abs(orc - ref)) <= 2 * R.U32 * np.max(np.abs(ref)) + 1e-12


@pytest.mark.parametrize("name", list(FILTERS))
def test_bound_is_tight(name):
    """the double-precision term of the bound stays far below the signal, so a wrong output cannot hide in it"""
    b, a = FILTERS[name]
    _, ref, bnd = R.bound(b, a, _stream(False), False)
    assert np.max(bnd - 2 * R.U32 * np.abs(ref)) <= 1e-6 * np.max(np.abs(ref))


@pytest.mark.parametrize("cplx", [False, True])
@pytest.mark.parametrize("name", list(FILTERS))
def test_model_within_bound(name, cplx):
    b, a = FILTERS[name]
    assert _run(b, a, cplx) <= 1.0


@pytest.mark.parametrize("mutant", MUTANTS)
@pytest.mark.parametrize("name", list(FILTERS))
def test_mutant_breaks_bound(name, mutant):
    b, a = FILTERS[name]
    if not R.mutant_applies(mutant, b, a):
        pytest.skip("the mutant cannot differ from the truth for this filter (iir_order_ref.mutant_applies)")
    assert _run(b, a, False, mutant) > 3.0
