"""CPU: the packed-weight cache (engine.WeightCache), `refresh_weights`, and the weight state that captured graphs and open decode
caches check (engine.WeightState): which weight updates each of them sees.  No kernel runs; `build` stands for the packing."""
import copy
import pickle

import pytest
import torch
import torch.nn as nn

from oracle import synth


class _Counter:
    def __init__(self):
        self.n = 0

    def __call__(self):
        self.n += 1
        return object()


class _FakeParam:
    """What the cache key reads from a parameter: storage address, version counter, device."""

    def __init__(self, ptr, version, device):
        self._ptr, self._version, self.device = ptr, version, device

    def data_ptr(self):
        return self._ptr


@pytest.fixture(autouse=True)
def _precision_reset():
    import vima_b200

    yield
    vima_b200.set_precision("f16x3")


def _tree():
    """Two levels of modules with a packed-weight cache each (the vima_b200.nn.Linear and build_mlp layouts)."""
    import vima_b200.nn as vnn

    torch.manual_seed(0)
    return nn.ModuleDict({"a": vnn.Linear(8, 4), "b": nn.Sequential(vnn.Linear(4, 4), nn.ModuleDict({"c": vnn.Linear(4, 2)}))})


def _fill(tree):
    """One cache entry per Linear in the tree, as a forward would leave them; returns the build counters."""
    counts = {}
    for name, m in tree.named_modules():
        if hasattr(m, "_wc"):
            counts[name] = _Counter()
            m._wc.get("w", (m.weight, m.bias), counts[name])
    return counts


def test_weight_cache_rebuilds_on_every_detectable_change():
    import vima_b200
    from vima_b200 import engine as eng

    wc = eng.WeightCache()
    w = nn.Parameter(torch.randn(4, 4))
    b = nn.Parameter(torch.zeros(4))
    build = _Counter()
    first = wc.get("w", (w, b), build)
    assert wc.get("w", (w, b), build) is first and build.n == 1          # plain re-call: no rebuild
    assert wc.get("w", (w, None), build) is not first and build.n == 2   # a different parameter set
    wc.get("w", (w, b), build)
    n = build.n
    with torch.no_grad():
        b.add_(1.0)                                                      # in-place under no_grad: version bump
    wc.get("w", (w, b), build)
    assert build.n == n + 1
    b2 = nn.Parameter(b.detach().clone())                                # a replaced tensor (same values, new storage)
    wc.get("w", (w, b2), build)
    assert build.n == n + 2
    wc.get("w", (w, b2), build)
    assert build.n == n + 2
    vima_b200.set_precision("f16f8")                                     # precision change
    wc.get("w", (w, b2), build)
    assert build.n == n + 3
    vima_b200.set_precision("f16x3")
    wc.get("w", (w, b2), build)
    assert build.n == n + 4


def test_weight_cache_key_includes_device():
    """Same address and version on another device is another weight (no second device here: the key reads three attributes)."""
    from vima_b200 import engine as eng

    wc = eng.WeightCache()
    build = _Counter()
    t = _FakeParam(4096, 0, "cuda:0")
    wc.get("w", (t,), build)
    wc.get("w", (t,), build)
    assert build.n == 1
    t.device = "cuda:1"
    wc.get("w", (t,), build)
    assert build.n == 2
    t._version = 1
    wc.get("w", (t,), build)
    assert build.n == 3


def test_weight_cache_sees_a_replacement_at_the_same_address():
    """Two replacements with no call in between: the second tensor can land in the block the first freed, at the same version.
    It is still another tensor, and the entry is rebuilt."""
    from vima_b200 import engine as eng

    wc = eng.WeightCache()
    build = _Counter()
    a = _FakeParam(8192, 0, "cuda:0")
    wc.get("w", (a, None), build)
    b = _FakeParam(8192, 0, "cuda:0")  # same address, same version, another tensor
    wc.get("w", (b, None), build)
    assert build.n == 2
    del a  # the first one is gone: its address is reused once more
    c = _FakeParam(8192, 0, "cuda:0")
    wc.get("w", (c, None), build)
    assert build.n == 3
    wc.get("w", (c, None), build)
    assert build.n == 3


def test_weight_cache_does_not_see_data_writes_refresh_does():
    """A write through `.data` moves no version counter: the cache keeps the old entry until refresh_weights."""
    import vima_b200

    tree = _tree()
    counts = _fill(tree)
    lin = tree["b"][0]
    lin.weight.data.copy_(torch.randn(4, 4))
    lin._wc.get("w", (lin.weight, lin.bias), counts["b.0"])
    assert counts["b.0"].n == 1  # the documented blind spot (INTEGRATION.md, weight updates)
    vima_b200.refresh_weights(tree)
    lin._wc.get("w", (lin.weight, lin.bias), counts["b.0"])
    assert counts["b.0"].n == 2


def test_refresh_weights_drops_every_entry_in_the_tree():
    import vima_b200

    tree = _tree()
    counts = _fill(tree)
    caches = {name: m._wc for name, m in tree.named_modules() if hasattr(m, "_wc")}
    assert sorted(caches) == ["a", "b.0", "b.1.c"]
    gens = {k: c.generation for k, c in caches.items()}
    vima_b200.refresh_weights(tree)
    for name, c in caches.items():
        assert c._store == {} and c.generation == gens[name] + 1, name
    _fill_counts = _fill(tree)
    assert all(v.n == 1 for v in _fill_counts.values())
    # a subtree only
    vima_b200.refresh_weights(tree["b"])
    assert caches["a"].generation == gens["a"] + 1 and caches["b.0"].generation == gens["b.0"] + 2


def test_policy_refresh_weights_reaches_every_cache():
    import vima_b200

    for pol in (vima_b200.VIMAPolicy(**synth.MODEL_CFGS["2M"]), vima_b200.VIMAGatoPolicy(**synth.GATO_CFGS["gato_tiny"])):
        caches = [m._wc for m in pol.modules() if "_wc" in m.__dict__]
        assert len(caches) >= 5
        for c in caches:
            c._store["x"] = ((), None)
        pol.refresh_weights()
        assert all(c._store == {} for c in caches)


def _updates():
    """(name, update(tree), seen) for every update route the weight state is meant to see -- and the one it cannot."""

    def load(tree):
        tree.load_state_dict({k: v + 1 for k, v in tree.state_dict().items()})

    def load_assign(tree):
        tree.load_state_dict({k: v + 1 for k, v in tree.state_dict().items()}, assign=True)

    def inplace(tree):
        with torch.no_grad():
            tree["b"][0].weight.mul_(2.0)

    def data_assign(tree):
        tree["b"][1]["c"].bias.data = torch.ones(2)

    def new_param(tree):
        tree["a"].weight = nn.Parameter(torch.randn(4, 8))

    def data_copy(tree):
        tree["a"].weight.data.copy_(torch.randn(4, 8))

    def data_copy_refresh(tree):
        import vima_b200

        data_copy(tree)
        vima_b200.refresh_weights(tree)

    return [("load_state_dict", load, True), ("load_state_dict_assign", load_assign, True), ("inplace_no_grad", inplace, True),
            ("data_assign", data_assign, True), ("new_parameter", new_param, True), ("data_copy", data_copy, False),
            ("data_copy_refresh", data_copy_refresh, True)]


@pytest.mark.parametrize("name,update,seen", _updates(), ids=[u[0] for u in _updates()])
def test_weight_state_sees_update_routes(name, update, seen):
    from vima_b200 import engine as eng

    tree = _tree()
    _fill(tree)
    st = eng.WeightState([tree])
    assert st.n_params() == 6 and st.changed() is None
    update(tree)
    assert (st.changed() is not None) == seen


def test_weight_state_holds_replaced_parameters():
    """The state keeps the parameters it recorded alive (a captured graph points at their storage)."""
    import weakref

    from vima_b200 import engine as eng

    tree = _tree()
    st = eng.WeightState([tree])
    old = weakref.ref(tree["a"].weight)
    tree["a"].weight = nn.Parameter(torch.randn(4, 8))
    assert old() is not None and st.changed() is not None
    del st
    assert old() is None


def test_record_weights_collects_owner_modules():
    """Inside `record_weights` every cache used is noted; the state covers all parameters of the owners (also the ones a kernel
    reads in fp32 without packing) and keeps the packed values."""
    from vima_b200 import engine as eng

    tree = _tree()
    extra = nn.Parameter(torch.zeros(3))  # a cache without an owner module contributes the parameters it was given
    loose = eng.WeightCache()
    with eng.record_weights() as weights:
        m = tree["b"][0]
        m._wc.get("w", (m.weight,), _Counter())
        m._wc.get("w", (m.weight,), _Counter())
        loose.get("x", (extra, None), _Counter())
    st = weights()
    assert st.n_params() == 2 + 1 and len(st._keep) == 3
    assert not eng._recorders
    tree["a"].weight = nn.Parameter(torch.randn(4, 8))  # not under the recorded owner
    assert st.changed() is None
    with torch.no_grad():
        tree["b"][0].bias.add_(1.0)  # under the owner, though the cache was given the weight only
    assert st.changed() is not None
    st = weights()
    with torch.no_grad():
        extra.add_(1.0)
    assert st.changed() is not None


def test_record_weights_collects_direct_reads():
    """Modules whose fp32 parameters go to a kernel without a cache (`engine.uses`) are recorded like cache owners; a state can
    also watch single (module, name) parameters."""
    from vima_b200 import engine as eng

    tree = _tree()
    with eng.record_weights() as weights:
        eng.uses(tree["b"][1]["c"])
        eng.uses(tree["b"][1]["c"])
    st = weights()
    assert st.n_params() == 2 and st.changed() is None
    tree["b"][1]["c"].weight = nn.Parameter(torch.randn(2, 4))
    assert st.changed() is not None
    one = eng.WeightState([tree["a"]], slots=[(tree["b"][0], "bias"), (tree["a"], "bias")])
    assert one.n_params() == 3
    with torch.no_grad():
        tree["b"][0].weight.add_(1.0)  # not watched
    assert one.changed() is None
    tree["b"][0].bias = nn.Parameter(torch.zeros(4))
    assert one.changed() is not None


def test_weight_cache_copy_and_pickle():
    """A deep copy's caches belong to the copy and start empty; pickling drops the packed weights."""
    tree = _tree()
    _fill(tree)
    cp = copy.deepcopy(tree)
    assert cp["a"]._wc.owner is cp["a"] and cp["a"]._wc._store == {}
    assert tree["a"]._wc.owner is tree["a"] and tree["a"]._wc._store != {}
    un = pickle.loads(pickle.dumps(tree))
    assert un["a"]._wc._store == {} and un["a"]._wc.owner is None


def test_decode_caches_refuse_changed_weights():
    """DecodeCache / SlotDecodeCache opened with a weight state refuse an append / step once it has changed (ValueError, before
    any state is touched), as they refuse another precision mode."""
    from vima_b200 import engine as eng
    from vima_b200.nn.xattn_gpt import DecodeCache, SlotDecodeCache, check_cache_append

    tree = _tree()
    p = eng.prec()
    dc = DecodeCache(B=2, Lmax=8, E=4, n_layer=1, device="cpu", split=True, precision=p.name, weights=eng.WeightState([tree]))
    sc = SlotDecodeCache(S=2, Lmax=8, Lp_cap=0, E=4, n_layer=1, device="cpu", split=True, precision=p.name, weights=eng.WeightState([tree]))
    check_cache_append(dc, 2, 3, 4, p)
    sc.check_step(2, 3, 4, p)
    tree.load_state_dict(tree.state_dict(), assign=False)
    with pytest.raises(ValueError, match="weights changed"):
        check_cache_append(dc, 2, 3, 4, p)
    with pytest.raises(ValueError, match="weights changed"):
        sc.check_step(2, 3, 4, p)
    with pytest.raises(ValueError, match="weights changed"):
        sc.check_precision(p)
    assert dc.L == 0
