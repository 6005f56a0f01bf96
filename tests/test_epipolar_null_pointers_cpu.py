"""Every epipolar attention entry point refuses a NULL required pointer with PS_ERR_INVALID_ARGUMENT (1) before it
touches a device: the forward, the atomic backward and the fixed-order backward, each input of ps_epipolar_inputs
(q_pe too, which is required when pe_dim > 0) and each of the entry point's own arguments.  ps_epipolar_geometry
refuses a NULL required pointer or a count below its minimum the same way, and a launch grid it cannot express
(b * v * (v - 1) > 65535 slices, grid_h * grid_w >= 2^31 rays) with PS_ERR_UNSUPPORTED (3).

The other pointers are a fake address, so the calls run in a child process that sees no GPU
(CUDA_VISIBLE_DEVICES=""): a check that stops refusing makes that call fail cleanly instead of launching a kernel
that would read the fake address."""
import json
import os
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
INPUTS = ["features", "segments", "valid", "rel_disparity", "q_feat", "q_pe"]
# entry point -> (its pointer arguments after (desc, inputs), the ones it requires at pe_dim > 0)
ENTRIES = {
    "ps_epipolar_attention_forward": (["z", "e", "mass", "lse"], ["z", "e", "lse"]),
    "ps_epipolar_attention_backward": (["lse", "dz", "de", "dmass", "d_row", "dq_feat", "dq_pe", "dbias", "dfeatures"],
                                       ["lse", "dz", "de", "d_row", "dq_feat", "dq_pe", "dfeatures"]),
    "ps_epipolar_attention_backward_deterministic": (
        ["lse", "dz", "de", "dmass", "d_row", "dq_feat", "dq_pe", "dbias", "dfeatures", "workspace"],
        ["lse", "dz", "de", "d_row", "dq_feat", "dq_pe", "dfeatures", "workspace"]),
}
CASES = [(entry, null) for entry, (_, required) in ENTRIES.items()
         for null in required + ["in." + n for n in INPUTS] + ["desc", "inputs"]]

CHILD = """
import ctypes, json, sys
from pixelsplat_b200 import _lib
entries, cases = json.loads(sys.argv[1]), json.loads(sys.argv[2])
FAKE = ctypes.c_void_p(0x1000)
out = []
for entry, null in cases:
    d = _lib.EpipolarDesc(1, 2, 4, 4, 8, 128, 2, 8)
    inp = _lib.EpipolarInputs(*([FAKE.value] * 7))
    if null.startswith("in."):
        setattr(inp, null[3:], None)
    args = [None if p == null else FAKE for p in entries[entry][0]]
    if entry.endswith("deterministic"):
        args.append(_lib.epipolar_backward_workspace_bytes(d))
    rc = getattr(_lib.lib, entry)(None if null == "desc" else ctypes.byref(d),
                                  None if null == "inputs" else ctypes.byref(inp), *args, None)
    out.append([rc, _lib.lib.ps_last_error().decode()])
print(json.dumps(out))
"""


@pytest.fixture(scope="module")
def results():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-c", CHILD, json.dumps(ENTRIES), json.dumps(CASES)], cwd=str(ROOT), env=env,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    return dict(zip(CASES, json.loads(r.stdout.strip().splitlines()[-1])))


@pytest.mark.parametrize("entry,null", CASES, ids=[f"{e[len('ps_epipolar_attention_'):]}-{n}" for e, n in CASES])
def test_rejects_a_null_required_pointer(results, entry, null):
    rc, err = results[(entry, null)]
    assert rc == 1, err


GEOMETRY_POINTERS = ["extrinsics", "intrinsics", "near_plane", "far_plane", "segments", "valid", "rel_disparity"]
# (batch, views, grid_h, grid_w, samples, NULL pointer or None) -> expected return code
GEOMETRY_CASES = {**{(1, 2, 4, 4, 8, p): 1 for p in GEOMETRY_POINTERS},
                  (0, 2, 4, 4, 8, None): 1, (1, 1, 4, 4, 8, None): 1, (1, 2, 0, 4, 8, None): 1,
                  (1, 2, 4, 0, 8, None): 1, (1, 2, 4, 4, 0, None): 1,
                  (1, 257, 4, 4, 8, None): 3, (2, 182, 4, 4, 8, None): 3, (65536, 2, 4, 4, 8, None): 3,
                  (1, 2, 65536, 32768, 8, None): 3, (1, 2, 46341, 46341, 8, None): 3}

GEOMETRY_CHILD = """
import ctypes, json, sys
from pixelsplat_b200 import _lib
names = json.loads(sys.argv[1])
FAKE = ctypes.c_void_p(0x1000)
out = []
for b, v, h, w, s, null in json.loads(sys.argv[2]):
    ptrs = [None if n == null else FAKE for n in names]
    rc = _lib.lib.ps_epipolar_geometry(b, v, h, w, s, *ptrs, FAKE, None)
    out.append([rc, _lib.lib.ps_last_error().decode()])
print(json.dumps(out))
"""


def test_geometry_refuses_before_enqueuing():
    cases = list(GEOMETRY_CASES)
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-c", GEOMETRY_CHILD, json.dumps(GEOMETRY_POINTERS), json.dumps(cases)],
                       cwd=str(ROOT), env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    got = json.loads(r.stdout.strip().splitlines()[-1])
    for case, (rc, err) in zip(cases, got):
        assert rc == GEOMETRY_CASES[case], (case, rc, err)
