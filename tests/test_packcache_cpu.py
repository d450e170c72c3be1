"""packcache: a pack is rebuilt exactly when a parameter or buffer of its module trees, the trees themselves or the
16-bit type change.  Plain nn modules on the CPU, no shared library."""
from __future__ import annotations

import copy

import pytest
import torch
from torch import nn

from hairfastgan_b200 import packcache


def _net():
    return nn.Sequential(nn.Conv2d(3, 4, 3), nn.BatchNorm2d(4),
                         nn.ModuleList([nn.Linear(4, 4), nn.Linear(4, 4)]),
                         nn.ModuleDict({"a": nn.Linear(4, 4)}), nn.ReLU())


class _Owner:
    """Counts the builds of one cache slot over ``roots``."""

    def __init__(self, *roots):
        self.roots = roots
        self.builds = 0

    def _build(self):
        self.builds += 1
        return object()

    def get(self, dtype=0):
        return packcache.get(self, "_pack", self.roots, dtype, self._build)


def _rebuilds(change, net=None) -> bool:
    net = _net() if net is None else net
    o = _Owner(net)
    o.get()
    o.get()
    assert o.builds == 1
    change(net)
    o.get()
    return o.builds == 2


def test_no_change_reuses_the_pack():
    assert not _rebuilds(lambda net: None)


def test_returns_the_stored_pack_and_its_key():
    net = _net()
    o = _Owner(net)
    p, k = o.get(dtype=7)
    assert o.get(dtype=7) == (p, k) and k == (packcache.key(net), 7)


@torch.no_grad()
def test_in_place_edit_rebuilds():
    assert _rebuilds(lambda net: net[0].weight.add_(1))
    assert _rebuilds(lambda net: net[1].running_mean.add_(1))


def test_load_state_dict_rebuilds():
    assert _rebuilds(lambda net: net.load_state_dict(_net().state_dict()))


def test_double_rebuilds_and_then_sees_buffer_edits():
    net = _net()
    assert _rebuilds(lambda n: n.double(), net)
    assert _rebuilds(lambda n: n[1].running_var.mul_(2), net)       # a buffer object .double() created


@pytest.mark.parametrize("replace", [
    lambda net: net.__setitem__(0, nn.Conv2d(3, 4, 3)),
    lambda net: net[2].__setitem__(1, nn.Linear(4, 4)),
    lambda net: net[3].__setitem__("a", nn.Linear(4, 4)),
    lambda net: setattr(net[2][0], "extra", nn.Linear(4, 4)),
], ids=["Sequential", "ModuleList", "ModuleDict", "setattr"])
def test_replaced_or_added_submodule_rebuilds(replace):
    assert _rebuilds(replace)


def test_new_buffer_or_parameter_rebuilds():
    assert _rebuilds(lambda net: net[0].register_buffer("extra", torch.zeros(2)))
    assert _rebuilds(lambda net: setattr(net[4], "extra", nn.Parameter(torch.zeros(2))))


def test_dtype_change_rebuilds():
    o = _Owner(_net())
    o.get(dtype=0)
    o.get(dtype=1)
    assert o.builds == 2


@torch.no_grad()
def test_rebuild_drops_captured_graphs():
    net = _net()
    o = _Owner(net)
    o.get()
    o._hf_graphs = {"sig": "graph"}
    o.get()
    assert o._hf_graphs
    net[0].weight.add_(1)
    o.get()
    assert "_hf_graphs" not in o.__dict__


def test_unrelated_module_neither_rebuilds_nor_rewalks():
    net = _net()
    o = _Owner(net)
    o.get()
    tree = packcache._trees[net]
    nn.Sequential(nn.Linear(2, 2), nn.ModuleList([nn.Conv2d(1, 1, 1)]))
    o.get()
    assert o.builds == 1 and packcache._trees[net] is tree


def test_deepcopy_packs_its_own_copy_and_sees_its_replacements():
    net = _net()
    o = _Owner(net)
    o.get()
    oc = copy.deepcopy(o)
    c = oc.roots[0]
    oc.get()
    assert oc.builds == 2 and o.builds == 1
    oc.get()
    assert oc.builds == 2
    c[2][0] = nn.Linear(4, 4)
    oc.get()
    o.get()
    assert oc.builds == 3 and o.builds == 1


def test_several_roots():
    a, b = _net(), _net()
    o = _Owner(a, b)
    o.get()
    b[2][1] = nn.Linear(4, 4)
    o.get()
    a[1].running_mean.add_(1)
    o.get()
    assert o.builds == 3
