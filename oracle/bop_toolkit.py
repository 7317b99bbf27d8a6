"""oracle/bop_toolkit.py -- load the BOP toolkit that the reference vendors (deps/bop_toolkit_challenge/bop_toolkit_lib).

TEST INFRASTRUCTURE ONLY, used to record the stored outputs tests/golden/reference/bop_eval_*.npz (MPX_RECORD_REFERENCE=1,
see tests/helpers.py: reference_outputs) where a checkout of the reference is named by $MEGAPOSE_REFERENCE, as
oracle/refload.py does for the reference's own package.  The toolkit's misc module imports pytz for its log timestamps
only; a stub stands in for it when pytz is absent.  Everything the tests record (pose_error, misc, pose_matching, score)
is the toolkit's own code, unmodified.
"""
from __future__ import annotations

import importlib
import os
import sys
import types
from pathlib import Path

TOOLKIT = (Path(os.environ["MEGAPOSE_REFERENCE"]).resolve() / "deps" / "bop_toolkit_challenge"
           if os.environ.get("MEGAPOSE_REFERENCE") else None)


def load() -> types.SimpleNamespace:
    """The toolkit's modules: misc, pose_error, pose_matching, score, visibility."""
    if TOOLKIT is None or not (TOOLKIT / "bop_toolkit_lib").is_dir():
        raise RuntimeError("no BOP toolkit: set MEGAPOSE_REFERENCE to a checkout of the reference")
    try:
        import pytz  # noqa: F401
    except ImportError:
        import datetime

        stub = types.ModuleType("pytz")
        stub.timezone = lambda name: datetime.timezone.utc
        sys.modules["pytz"] = stub
    if str(TOOLKIT) not in sys.path:
        sys.path.insert(0, str(TOOLKIT))
    names = ("misc", "pose_error", "pose_matching", "score", "visibility")
    return types.SimpleNamespace(**{n: importlib.import_module(f"bop_toolkit_lib.{n}") for n in names})
