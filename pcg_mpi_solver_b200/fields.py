"""Strains and stresses of a hex box recovered on the device from its displacement (csrc/fields.cuh, pcgb_fields_*): element
strain and stress, principal stresses and strains, and their nodal averages, on one rank or across ranks.  They stand in for
the reference's updateElemStrain (pcg_solver.py:601-618), getPrincipalStress / getPrincipalStrain (file_operations.py:251-301)
and getNodalPS (pcg_solver.py:730-814) on the boxes `hexmesh` generates (uniform or a voxel field of Young's moduli).

    op = generate_box_operator(block, E_field=f);  ...solve for x...
    F = HexFields(block, E_field=f)
    F.element(x)["stress"]        # (ne, 6): Voigt 11, 22, 33, 23, 13, 12 per element, e = (z * ne[1] + y) * ne[0] + x
    F.nodal(x, "stress")          # (nodes, 3): P1 >= P2 >= P3 averaged at every node of the box, clamped line included

The arithmetic (centroid Q1 gradient, the stress law of hex_element_stiffness, the invariant-form principal values and
the fixed nodal summation order) is stated in the header of csrc/fields.cuh and in DESIGN §2.10.

`PeriodicFields(cell, E_field=f)` does the same for a periodic cell (hexmesh.PeriodicCell, DESIGN §2.13) from its
fluctuation u~ and a macroscopic strain: `element(x, strain)` and the bit-reproducible volume average `average(x, strain)`.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from . import _lib
from .hexmesh import HexBlock, PeriodicCell, _same_device, check_field, interface_node_lists

ELEMENT_FIELDS = {"strain": 6, "stress": 6, "ps": 3, "pe": 3}


class HexFields:
    """Field recovery of `block` on `device`.  E_field: one Young's modulus per element (shape (ne[2], ne[1], ne[0]), as
    generate_matrix takes it), replacing block.E; kept on the device for the object's lifetime (8 bytes per element).
    Across ranks pass the communicator and the partition (`blocks`, with block is blocks[comm.rank]): the constructor then
    builds the node-level halo plan once, collectively, so every rank must construct its HexFields together."""

    def __init__(self, block: HexBlock, device="cuda", E_field=None, comm=None, blocks=None):
        if (comm is None) != (blocks is None):
            raise ValueError("HexFields: comm and blocks go together")
        if blocks is not None and block is not blocks[comm.rank]:
            raise ValueError("HexFields: block must be blocks[comm.rank]")
        self.block = block
        self.device = torch.device(device) if comm is None else comm.device
        self.n_elements = int(np.prod(block.ne))
        self.n_nodes = int(np.prod([v + 1 for v in block.ne]))
        self._E = None
        if E_field is not None:
            check_field(E_field, block, self.device)
            t = torch.from_numpy(E_field) if isinstance(E_field, np.ndarray) else E_field
            self._E = t.reshape(-1).to(self.device, torch.float64).contiguous()
        self._h = ctypes.c_void_p()
        self._halo = None
        lib = _lib.load()
        box = block.cbox()
        with torch.cuda.device(self.device):
            _lib.check(lib.pcgb_fields_create(ctypes.byref(box), float(block.h), float(block.E), float(block.nu), _lib.ptr(self._E),
                                              ctypes.byref(self._h)), "pcgb_fields_create")
            if comm is not None:
                from .solver import make_halo
                nbr, lists = interface_node_lists(blocks, comm.rank)
                lists4 = [(4 * v[:, None] + np.arange(4)[None, :]).ravel() for v in lists]
                self._halo = make_halo(comm, nbr, lists4, 4 * self.n_nodes)

    def _check_x(self, x: torch.Tensor):
        if not isinstance(x, torch.Tensor) or x.dtype != torch.float64 or x.dim() != 1 or x.numel() != self.block.n:
            raise ValueError(f"HexFields: x must be a float64 vector of the box's {self.block.n} free dofs")
        if x.device.type != "cuda" or not _same_device(x.device, self.device):
            raise ValueError(f"HexFields: x is on {x.device}, expected {self.device}")
        return x.contiguous()

    def element(self, x: torch.Tensor, fields=("strain", "stress", "ps", "pe")) -> dict:
        """The element fields named in `fields` from one pass over the box: 'strain' and 'stress' (ne, 6), 'ps' (principal
        stresses) and 'pe' (principal strains) (ne, 3), float64 device tensors."""
        x = self._check_x(x)
        bad = [f for f in fields if f not in ELEMENT_FIELDS]
        if bad or not fields:
            raise ValueError(f"HexFields.element: fields must be a non-empty subset of {tuple(ELEMENT_FIELDS)}, got {tuple(fields)}")
        out = {f: torch.empty((self.n_elements, ELEMENT_FIELDS[f]), dtype=torch.float64, device=self.device) for f in fields}
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().pcgb_fields_element(self._h, _lib.ptr(x), *(_lib.ptr(out.get(f)) for f in ELEMENT_FIELDS),
                                                       _lib.stream_ptr()), "pcgb_fields_element")
        return out

    def nodal(self, x: torch.Tensor, kind: str = "stress") -> torch.Tensor:
        """Principal stresses (kind 'stress') or strains ('strain') averaged at every node of the box, (nodes, 3), node =
        (lz * (ne[1] + 1) + ly) * (ne[0] + 1) + lx; across ranks the interface nodes average over every rank's elements."""
        if kind not in ("stress", "strain"):
            raise ValueError(f"HexFields.nodal: kind must be 'stress' or 'strain', got {kind!r}")
        x = self._check_x(x)
        work = torch.empty(4 * self.n_nodes, dtype=torch.float64, device=self.device)
        out = torch.empty((self.n_nodes, 3), dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().pcgb_fields_nodal(self._h, _lib.ptr(x), 0 if kind == "stress" else 1, self._halo, _lib.ptr(work),
                                                     _lib.ptr(out), _lib.stream_ptr()), "pcgb_fields_nodal")
        return out

    def __del__(self):
        try:
            lib = _lib.load()
            if self._h:
                lib.pcgb_fields_destroy(self._h)
                self._h = ctypes.c_void_p()
            if self._halo:
                lib.pcgb_halo_destroy(self._halo)
                self._halo = None
        except Exception:
            pass


def _voigt_strain(strain) -> np.ndarray:
    e = np.ascontiguousarray(strain, dtype=np.float64)
    if e.shape != (6,) or not np.isfinite(e).all():
        raise ValueError(f"PeriodicFields: strain must be 6 finite Voigt components, got {strain!r}")
    return e


class PeriodicFields:
    """Field recovery of a periodic cell on `device`.  x is the periodic fluctuation u~ (3 ne[0] ne[1] ne[2] dofs, the
    numbering of hexmesh.generate_periodic_operator) and `strain` the macroscopic strain (Voigt 11, 22, 33, 23, 13, 12 with
    engineering shears), added to every element's centroid strain.  E_field: as HexFields, kept on the device."""

    def __init__(self, cell: PeriodicCell, device="cuda", E_field=None):
        self.block = cell
        self.device = torch.device(device)
        self.n_elements = cell.n_elements
        self._E = None
        if E_field is not None:
            check_field(E_field, cell, self.device)
            t = torch.from_numpy(E_field) if isinstance(E_field, np.ndarray) else E_field
            self._E = t.reshape(-1).to(self.device, torch.float64).contiguous()
        self._h = ctypes.c_void_p()
        box = cell.cbox()
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().pcgb_fields_create_periodic(ctypes.byref(box), float(cell.h), float(cell.E), float(cell.nu),
                                                               _lib.ptr(self._E), ctypes.byref(self._h)), "pcgb_fields_create_periodic")

    def _check_x(self, x: torch.Tensor):
        if not isinstance(x, torch.Tensor) or x.dtype != torch.float64 or x.dim() != 1 or x.numel() != self.block.n:
            raise ValueError(f"PeriodicFields: x must be a float64 vector of the cell's {self.block.n} dofs")
        if x.device.type != "cuda" or not _same_device(x.device, self.device):
            raise ValueError(f"PeriodicFields: x is on {x.device}, expected {self.device}")
        return x.contiguous()

    def element(self, x: torch.Tensor, strain, fields=("strain", "stress", "ps", "pe")) -> dict:
        """HexFields.element's outputs with the macroscopic strain included (strain and stress with tensor shears)."""
        x = self._check_x(x)
        e = _voigt_strain(strain)
        bad = [f for f in fields if f not in ELEMENT_FIELDS]
        if bad or not fields:
            raise ValueError(f"PeriodicFields.element: fields must be a non-empty subset of {tuple(ELEMENT_FIELDS)}, got {tuple(fields)}")
        out = {f: torch.empty((self.n_elements, ELEMENT_FIELDS[f]), dtype=torch.float64, device=self.device) for f in fields}
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().pcgb_fields_element_periodic(self._h, _lib.ptr(x), e.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                                                                *(_lib.ptr(out.get(f)) for f in ELEMENT_FIELDS), _lib.stream_ptr()),
                       "pcgb_fields_element_periodic")
        return out

    def average(self, x: torch.Tensor, strain):
        """(<strain>, <stress>): the volume averages over the cell, two float64 numpy arrays of 6 (Voigt, tensor shears),
        from one element pass and a fixed-order reduction (csrc/fields.cuh), bit-reproducible from run to run."""
        x = self._check_x(x)
        e = _voigt_strain(strain)
        es, ss = np.empty(6), np.empty(6)
        dp = ctypes.POINTER(ctypes.c_double)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().pcgb_fields_average(self._h, _lib.ptr(x), e.ctypes.data_as(dp), es.ctypes.data_as(dp),
                                                       ss.ctypes.data_as(dp), _lib.stream_ptr()), "pcgb_fields_average")
        return es, ss

    def nodal(self, x=None, kind: str = "stress"):
        raise ValueError("PeriodicFields.nodal: nodal averages on periodic cells are not implemented")

    def __del__(self):
        try:
            if self._h:
                _lib.load().pcgb_fields_destroy(self._h)
                self._h = ctypes.c_void_p()
        except Exception:
            pass
