"""Static unit plan: how a model's parameters are grouped, flattened and sharded.

This replaces the reference's *traced* execution order (``partitioned_param_coordinator.py:235``
learns the module order from the first iteration) with a plan computed once from the module tree:

* a **unit** is the granularity of gather / release / reduce -- by default every element of an
  ``nn.ModuleList`` with more than one element (i.e. one transformer block) and every remaining
  top-level parameter-bearing subtree;
* inside a unit the parameters are laid out back to back (16-byte aligned) in ONE flat buffer
  whose length is padded to ``world * SHARD_ALIGN``; rank ``r`` owns the contiguous slice
  ``[r*S, (r+1)*S)``.  ``all_gather_into_tensor`` therefore lands directly in the layout the
  parameter views use and ``reduce_scatter_tensor`` consumes the gradient views with no
  interleave/copy step (the reference needs ``torch.cat`` + ``narrow`` on both paths,
  ``partition_parameters.py:1183``, ``coalesced_collectives.py:198``).

Everything in this file is pure bookkeeping (no collectives, no CUDA) and is unit-tested on CPU.
"""
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import torch
from torch import nn

PARAM_ALIGN = 8  # elements: 16 bytes for bf16/fp16, 32 bytes for fp32 -> every view is vector-aligned
SHARD_ALIGN = 128  # elements per rank granularity


def _round_up(x, m):
    return (x + m - 1) // m * m


@dataclass
class ParamSlot:
    param: nn.Parameter
    name: str
    offset: int  # element offset inside the unit flat buffer
    numel: int
    shape: torch.Size
    group: int = 0  # optimizer param-group index


@dataclass
class Unit:
    index: int
    name: str
    module: Optional[nn.Module]
    slots: List[ParamSlot] = field(default_factory=list)
    full_numel: int = 0  # padded
    shard_numel: int = 0
    arena_offset: int = 0  # offset of this unit's shard inside the rank-local shard arena
    persistent: bool = False
    # modules outside the unit's subtree that hold one of its parameters directly (a tied LM head): (name, module)
    borrowers: List[Tuple[str, nn.Module]] = field(default_factory=list)

    @property
    def raw_numel(self):
        return sum(s.numel for s in self.slots)

    def shard_range(self, rank: int) -> Tuple[int, int]:
        return rank * self.shard_numel, (rank + 1) * self.shard_numel


def default_unit_modules(model: nn.Module, leaf_classes: Sequence[type] = ()) -> List[Tuple[str, nn.Module]]:
    """Choose unit roots: ModuleList elements (len > 1), user-marked leaf modules, else top-level
    parameter-bearing children; parameters owned directly by ``model`` form a final root unit."""
    from deepspeed_b200.utils.z3_leaf_module import z3_leaf_module
    units: List[Tuple[str, nn.Module]] = []

    def has_params(m):
        return any(True for _ in m.parameters())

    def visit(prefix: str, m: nn.Module):
        if z3_leaf_module(m) or (leaf_classes and isinstance(m, tuple(leaf_classes))):
            units.append((prefix, m))
            return
        if isinstance(m, (nn.ModuleList, nn.Sequential)) and len(m) > 1:
            for i, child in enumerate(m):
                if has_params(child):
                    visit(f"{prefix}.{i}" if prefix else str(i), child)
            return
        # does any descendant contain a multi-element ModuleList / leaf?  then recurse
        nested = any((isinstance(c, (nn.ModuleList, nn.Sequential)) and len(c) > 1) or z3_leaf_module(c)
                     for c in m.modules() if c is not m)
        if nested:
            own = [p for p in m.parameters(recurse=False)]
            if own:
                units.append((prefix + ":own" if prefix else ":own", m))
            for cname, child in m.named_children():
                if has_params(child):
                    visit(f"{prefix}.{cname}" if prefix else cname, child)
        else:
            units.append((prefix, m))

    visit("", model)
    return units


def build_units(model: nn.Module,
                world: int,
                param_to_group: Optional[Dict[int, int]] = None,
                persistence_threshold: int = 0,
                max_unit_numel: Optional[int] = None,
                leaf_classes: Sequence[type] = (),
                trainable_only: bool = False,
                param_filter=None) -> List[Unit]:
    """Build the unit plan for ``model``.  Shared (tied) parameters are assigned to the first unit
    that references them; every other module holding one directly is recorded as a borrower of that
    unit (:attr:`Unit.borrowers`).  Units larger than ``max_unit_numel`` are not split (a unit is the
    module-hook granularity) but the value is used by ZeRO-1/2 to form reduce buckets."""
    param_to_group = param_to_group or {}
    roots = default_unit_modules(model, leaf_classes)
    names = {id(p): n for n, p in model.named_parameters(remove_duplicate=False)}
    seen = set()
    units: List[Unit] = []
    for uname, mod in roots:
        own_only = uname.endswith(":own")
        plist = list(mod.named_parameters(recurse=not own_only, remove_duplicate=True))
        slots = []
        off = 0
        for local_name, p in plist:
            if id(p) in seen:
                continue
            if trainable_only and not p.requires_grad:
                continue
            if param_filter is not None and not param_filter(p):
                continue
            seen.add(id(p))
            numel = _ds_numel(p)
            slots.append(
                ParamSlot(param=p,
                          name=names.get(id(p), f"{uname}.{local_name}"),
                          offset=off,
                          numel=numel,
                          shape=_ds_shape(p),
                          group=param_to_group.get(id(p), 0)))
            off = _round_up(off + numel, PARAM_ALIGN)
        if not slots:
            continue
        u = Unit(index=len(units), name=uname or "root", module=None if own_only else mod, slots=slots)
        u.full_numel = _round_up(max(off, 1), world * SHARD_ALIGN)
        u.shard_numel = u.full_numel // world
        u.persistent = u.raw_numel <= persistence_threshold
        units.append(u)
    arena = 0
    for u in units:
        u.arena_offset = arena
        arena += u.shard_numel
    _find_borrowers(model, units, roots)
    return units


def _find_borrowers(model: nn.Module, units: List[Unit], roots) -> None:
    root_of = dict(roots)  # a ":own" unit holds its root module's own parameters: that module is its subtree
    subtree = {u.index: {id(m) for m in ([root_of[u.name]] if u.module is None else u.module.modules())} for u in units}
    owner = {id(s.param): u for u in units for s in u.slots}
    for name, m in model.named_modules():
        for p in m.parameters(recurse=False):
            u = owner.get(id(p))
            if u is not None and id(m) not in subtree[u.index] and all(b is not m for _, b in u.borrowers):
                u.borrowers.append((name, m))


def _ds_numel(p):
    return int(getattr(p, "ds_numel", p.numel()))


def _ds_shape(p):
    return getattr(p, "ds_shape", p.shape)


@dataclass
class Segment:
    """A run of the rank-local arena whose elements share one optimizer param group."""
    group: int
    start: int
    end: int


def arena_segments(units: List[Unit], rank: int) -> List[Segment]:
    """Intersect every parameter with this rank's shard and emit arena-coordinate segments,
    merging neighbours of the same group.  Alignment padding is attached to the preceding
    parameter's segment (padding holds zeros and zero gradients, so the update is a no-op)."""
    raw: List[Segment] = []
    for u in units:
        lo, hi = u.shard_range(rank)
        pieces = []
        for s in u.slots:
            a, b = max(s.offset, lo), min(s.offset + s.numel, hi)
            if a < b:
                pieces.append([a, b, s.group])
        if not pieces:  # this rank's slice of the unit is pure padding
            pieces = [[lo, hi, u.slots[-1].group]]
        pieces[0][0] = lo
        for i in range(len(pieces) - 1):
            pieces[i][1] = pieces[i + 1][0]
        pieces[-1][1] = hi
        for a, b, g in pieces:
            raw.append(Segment(g, u.arena_offset + a - lo, u.arena_offset + b - lo))
    merged: List[Segment] = []
    for s in raw:
        if merged and merged[-1].group == s.group and merged[-1].end == s.start:
            merged[-1].end = s.end
        else:
            merged.append(Segment(s.group, s.start, s.end))
    return merged


def param_fragments(unit: Unit, slot: ParamSlot, world: int) -> List[Tuple[int, int, int, int]]:
    """For one parameter return ``(rank, param_start, arena_start, length)`` pieces describing which
    part of the parameter lives where (the analogue of the reference ``tensor_fragment`` mapping,
    ``utils/tensor_fragment.py:312``)."""
    out = []
    for r in range(world):
        lo, hi = unit.shard_range(r)
        a, b = max(slot.offset, lo), min(slot.offset + slot.numel, hi)
        if a < b:
            out.append((r, a - slot.offset, unit.arena_offset + (a - lo), b - a))
    return out
