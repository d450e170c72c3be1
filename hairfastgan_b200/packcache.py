"""The one cache rule for weights packed into kernel layouts.

Every network here packs its parameters once (folded BatchNorm, 16-bit, K-major, lookup tables), keeps the pack on a
module and packs again when a weight changes.  ``get`` reuses a pack while the key of its module trees and the 16-bit
type it was packed for are unchanged.  The key is (storage pointer, version counter) of every parameter and buffer,
read through each module's live ``_parameters`` / ``_buffers`` dicts, so in-place edits and ``load_state_dict`` (the
version) and ``.to()`` / ``.double()`` (new storage, new buffer objects) change it on any module class, with no hook
on the class.

Walking a 600-module encoder costs as much as its kernels at swap()'s batch sizes, so live views of the non-empty
dicts are kept per root (outside the module: a ``copy.deepcopy`` of a packed network is walked afresh).  They are
rebuilt when a submodule, parameter or buffer is registered on a module of a cached tree; an empty dict only changes
through such a registration.
"""
from __future__ import annotations

import weakref

from torch.nn.modules import module as _module

_trees = weakref.WeakKeyDictionary()   # root -> (epoch, views of its non-empty _parameters / _buffers)
_walked = weakref.WeakSet()            # every module of every cached tree
_epoch = 0                             # bumped by each registration on one of them


def _on_register(module, name, value):
    global _epoch
    if module in _walked:
        _epoch += 1


_module.register_module_module_registration_hook(_on_register)
_module.register_module_parameter_registration_hook(_on_register)
_module.register_module_buffer_registration_hook(_on_register)


def _views(root) -> list:
    tree = _trees.get(root)
    if tree is None or tree[0] != _epoch:
        mods = list(root.modules())
        _walked.update(mods)
        tree = _trees[root] = (_epoch, [d.values() for m in mods for d in (m._parameters, m._buffers) if d])
    return tree[1]


def key(*roots) -> tuple:
    """(data_ptr, _version) of every parameter and buffer under ``roots``."""
    return tuple([(t.data_ptr(), t._version) for root in roots for v in _views(root) for t in v if t is not None])


def get(owner, slot: str, roots, dtype, build):
    """``(pack, key)``: the pack stored in ``owner.__dict__[slot]`` while ``(key(*roots), dtype)`` is unchanged,
    otherwise ``build()``'s result, stored there.  A rebuild drops the owner's captured CUDA graphs (graphs.py), which
    replay the old pack.  While unchanged the stored key object is returned, so comparing it with the key a graph was
    captured under is an identity check."""
    k = (key(*roots), dtype)
    hit = owner.__dict__.get(slot)
    if hit is not None and hit[0] == k:
        return hit[1], hit[0]
    pack = build()
    owner.__dict__[slot] = (k, pack)
    owner.__dict__.pop("_hf_graphs", None)
    return pack, k
