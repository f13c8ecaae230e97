"""The binding's shared lifetime code (dmosopt_b200/_lib.py): the owner of every library object and the mirrored
read-only outputs of the optimizer generators past the page-locked budget."""

import ctypes
import gc
import weakref

import numpy as np
import pytest

from dmosopt_b200 import _lib

OWNERS = [("GPHandle", "dmo_gp_destroy"), ("MTGPHandle", "dmo_mtgp_destroy"), ("SVGPHandle", "dmo_svgp_destroy"),
          ("DGPHandle", "dmo_dgp_destroy"), ("SVGPFitState", "dmo_svgp_fit_destroy"), ("DGPFitState", "dmo_dgp_fit_destroy"),
          ("FeasModel", "dmo_feas_destroy")]


class _StubLibrary:
    """Records every library call instead of making it."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        return lambda *args: self.calls.append((name,) + args) or 0


def _owner_calls(cls_name, ctx):
    """The library calls that one owner with a dummy handle makes across close(); close(); del, with ``ctx`` as the main
    context.  Objects collected meanwhile may call the stub as well: only the calls with this owner's handle count."""
    gc.collect()  # earlier tests' garbage is released through the real library, not the stub
    cls = getattr(_lib, cls_name)
    assert issubclass(cls, _lib._LibObject)
    stub = _StubLibrary()
    owner = cls.__new__(cls)  # no create call: the handle is a dummy the stub alone sees
    h = owner._h = ctypes.c_void_p(0x5EED000)
    alive = weakref.ref(owner)
    mp = pytest.MonkeyPatch()
    mp.setattr(_lib, "_lib", stub)
    mp.setattr(_lib, "_ctx", ctx)
    try:
        owner.close()
        owner.close()
        del owner
    finally:
        leaked = alive()
        if leaked is not None:
            leaked._h = None  # the dummy handle never reaches the real library
        mp.undo()
    assert leaked is None
    return [c for c in stub.calls if len(c) == 3 and c[2] is h], h


@pytest.mark.parametrize("cls_name,destroy", OWNERS)
def test_owner_destroys_its_object_exactly_once(cls_name, destroy):
    ctx = object()
    calls, h = _owner_calls(cls_name, ctx)
    assert calls == [(destroy, ctx, h)]


@pytest.mark.parametrize("cls_name,destroy", OWNERS)
def test_owner_destroys_nothing_without_the_main_context(cls_name, destroy):
    calls, _ = _owner_calls(cls_name, None)
    assert calls == []


def _served_from_mirror_past_budget(monkeypatch, generate):
    """generate() under a page-locked budget of zero: the same values as under the default budget, no page-locked bytes
    taken, the device copy still registered as its mirror and dropped with the array."""
    expected = np.array(generate())
    gc.collect()
    monkeypatch.setattr(_lib, "_PIN_LIVE_LIMIT", 0)
    live = _lib._pin_live_bytes
    x = generate()
    assert _lib._pin_live_bytes <= live, "the output was page-locked past the budget"
    assert not x.flags.writeable and np.array_equal(x, expected)
    m = _lib.mirror_ptr(x)
    assert m is not None, "the output is not served from its device copy"
    back = np.empty_like(x)
    _lib.memcpy(back, m, x.nbytes)
    assert np.array_equal(back, expected)
    addr = x.ctypes.data
    del x
    gc.collect()
    assert addr not in _lib._mirrors


@pytest.mark.gpu
def test_smpso_generate_past_the_page_locked_budget(monkeypatch):
    _lib.context()
    rng = np.random.default_rng(5)
    swarms, pop, d = 3, 40, 6
    lb, ub = -rng.random(d), 1.0 + rng.random(d)
    n = swarms * pop
    parm = (lb + rng.random((n, d)) * (ub - lb)).astype(np.float32).astype(np.float64)
    vel = rng.standard_normal((n, d)) * (ub - lb) * 0.3
    obj = rng.random((n, 2)).astype(np.float32).astype(np.float64)
    sw = _lib.SmpsoSwarms(parm, obj, vel, swarms, pop)
    _served_from_mirror_past_budget(monkeypatch, lambda: sw.generate(np.full(d, 20.0), lb, ub, 1.0 / d, 17, 2))


@pytest.mark.gpu
def test_cmaes_generate_past_the_page_locked_budget(monkeypatch):
    _lib.context()
    rng = np.random.default_rng(6)
    npar, n, d = 5, 64, 7
    px = rng.random((npar, d)) - 0.5
    sig = rng.random(npar) * 0.05 + 0.01
    A = _lib.resident_rows(np.eye(d)[None] + 0.1 * rng.standard_normal((npar, d, d)))
    pidx = rng.integers(0, npar, size=n)
    z = rng.standard_normal((n, d))
    lb, ub = -1.0 - rng.random(d), 1.0 + rng.random(d)
    _served_from_mirror_past_budget(monkeypatch, lambda: _lib.cmaes_generate(px, sig, A, pidx, z, lb, ub))
