"""Generates tests/golden/ply_export_v1.npz by running the REFERENCE's export_ply (src/model/ply_export.py) on the
CPU.  Authoring container only:

    python oracle/make_ply_golden.py

TEST INFRASTRUCTURE.  plyfile is absent offline; oracle/_stubs/plyfile hands the structured vertex array back
instead of writing a file.  Everything else is the reference's own code (scipy quaternions included).  Inputs are
regenerated from tests/ply_util.py on both sides; only the reference's records are stored, as float32 [n, 17] per
case, with the property names in file order.
"""
from __future__ import annotations

import sys
import tempfile
import types
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
REFERENCE = Path("/root/reference")
sys.path.insert(0, str(ROOT))
from tests import ply_util  # noqa: E402

OUT = ROOT / "tests" / "golden" / "ply_export_v1.npz"


def load_export_ply():
    for p in (str(ROOT / "oracle" / "_stubs"), str(REFERENCE)):
        if p not in sys.path:
            sys.path.insert(0, p)
    if "src.model" not in sys.modules:          # its encoder / decoder packages are not needed
        m = types.ModuleType("src.model")
        m.__path__ = [str(REFERENCE / "src" / "model")]
        sys.modules["src.model"] = m
    from plyfile import PlyData
    from src.model.ply_export import export_ply
    return export_ply, PlyData


def main() -> None:
    export_ply, PlyData = load_export_ply()
    out = {}
    tmp = tempfile.TemporaryDirectory()          # export_ply creates the parent directory of its path
    for name, _, n in ply_util.PLY_CASES:
        c = ply_util.ply_case(name)
        PlyData.written.clear()
        export_ply(c["extrinsics"], c["means"], c["scales"], c["rotations"], c["harmonics"], c["opacities"],
                   Path(tmp.name) / f"{name}.ply")
        (_, vertex), = PlyData.written
        names = list(vertex.dtype.names)
        assert len(vertex) == n and all(vertex.dtype[k] == np.dtype("f4") for k in names)
        out[name] = np.stack([vertex[k] for k in names], axis=-1)
        out["names"] = np.array(names)
    tmp.cleanup()
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT} ({OUT.stat().st_size} bytes): " + ", ".join(f"{k} {v.shape}" for k, v in out.items()))


if __name__ == "__main__":
    main()
