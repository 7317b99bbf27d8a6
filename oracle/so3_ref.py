"""oracle/so3_ref.py -- SO(3) grid for the CPU oracle (TEST INFRASTRUCTURE ONLY).

Restates load_SO3_grid (src/megapose/utils/transform_utils.py:27-50).  Where a checkout of the reference is named by
$MEGAPOSE_REFERENCE (oracle/refload.py) the quaternions are parsed from the reference's own text file; elsewhere from the
converted data asset (tests/test_oracle_vs_reference.py checks the asset against what the reference's file gives).
"""
from __future__ import annotations

from pathlib import Path

import numpy as np
import torch

from .lib3d_ref import unitquat_to_rotmat
from .refload import REF_ROOT

_REF = REF_ROOT / "data" if REF_ROOT is not None else None
_ASSET = Path(__file__).resolve().parents[1] / "megapose6d_b200" / "data"


def load_quats(resolution: int) -> torch.Tensor:
    ref = _REF / f"data_{resolution}.qua" if _REF is not None else None
    if ref is not None and ref.is_file():
        quats = [[float(v) for v in line.split()] for line in ref.read_text().splitlines() if line.strip()]
        return torch.tensor(quats)
    return torch.tensor(np.load(_ASSET / f"so3_grid_{resolution}.npy").tolist())


def load_SO3_grid_reference(resolution: int) -> torch.Tensor:
    return unitquat_to_rotmat(load_quats(resolution))
