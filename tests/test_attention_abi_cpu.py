"""The ViT attention and the 256-token self-attention entry points refuse what their kernels cannot run, before they
touch a device: a NULL pointer, a shape out of range (tokens, heads, dim_head, n_images), a pointer that is not
16-byte aligned, a short workspace, and for the self-attention a negative or non-finite scale (its forward takes the
row max on unscaled logits, so a negative scale would overflow exp2).  Refusals are PS_ERR_INVALID_ARGUMENT (1) for a
bad argument and PS_ERR_UNSUPPORTED (3) for a shape the kernels are not written for; n_images > 65535 does not fit
grid.z.

The pointers are fake addresses, so the calls run in a child process that sees no GPU (CUDA_VISIBLE_DEVICES=""): a
check that stops refusing makes that call fail cleanly instead of launching a kernel that would read them."""
import json
import math
import os
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]

# entry point -> its pointer arguments; the cases below are (id, entry, (n, tokens, heads, dim_head), scale,
# {pointer: fake address, 0 for NULL}, workspace bytes or None for enough, expected return code)
VIT_PTRS = {"ps_vit_attention_forward": ["qkv", "out", "lse"],
            "ps_vit_attention_backward": ["qkv", "out", "d_out", "lse", "d_qkv", "workspace"],
            "ps_self_attention_forward": ["qkv", "out"],
            "ps_self_attention_forward_stats": ["qkv", "out", "stats"],
            "ps_self_attention_backward": ["qkv", "out", "d_out", "stats", "d_qkv"]}
VIT_OK, SA_OK = (2, 65, 6, 64), (2, 256, 4, 128)


def _cases():
    cases = []
    for entry, names in VIT_PTRS.items():
        ok = VIT_OK if "vit" in entry else SA_OK
        for p in names:
            cases.append((f"{entry}-null-{p}", entry, ok, 0.125, {p: 0}, None, 1))
        for p in names:
            if p not in ("lse", "workspace", "stats"):
                cases.append((f"{entry}-misaligned-{p}", entry, ok, 0.125, {p: 0x1004}, None, 1))
        n, L, h, d = ok
        bad = [((0, L, h, d), 1), ((n, L, 0, d), 1), ((n, L, 17, d), 1 if "self" in entry else 3),
               ((65536, L, h, d), 3), ((n, L, h, d // 2), 3), ((n, L, h, d * 2), 3)]
        if "vit" in entry:
            bad += [((n, 0, h, d), 1), ((n, 16385, h, d), 3)]
        else:
            bad += [((n, 255, h, d), 3), ((n, 257, h, d), 3)]
        for shape, rc in bad:
            cases.append((f"{entry}-shape-{'x'.join(map(str, shape))}", entry, shape, 0.125, {}, None, rc))
        if "self" in entry:
            for s in (-0.125, -1e-30, math.inf, -math.inf, math.nan):
                cases.append((f"{entry}-scale-{s}", entry, ok, s, {}, None, 1))
        if entry == "ps_vit_attention_backward":
            need = VIT_OK[0] * VIT_OK[1] * VIT_OK[2] * 4
            cases.append((f"{entry}-short-workspace", entry, ok, 0.125, {}, need - 1, 1))
    return cases


CASES = _cases()

CHILD = """
import ctypes, json, sys
from pixelsplat_b200 import _lib
ptrs, cases = json.loads(sys.argv[1]), json.loads(sys.argv[2])
out = []
for _, entry, (n, L, h, d), scale, over, ws, _ in cases:
    p = [ctypes.c_void_p(over.get(name, 0x1000) or None) for name in ptrs[entry]]
    f = getattr(_lib.lib, entry)
    s = ctypes.c_float(scale)
    if entry == "ps_vit_attention_forward":
        rc = f(n, L, h, d, p[0], s, p[1], p[2], None)
    elif entry == "ps_vit_attention_backward":
        rc = f(n, L, h, d, p[0], p[1], p[2], p[3], s, p[4], p[5], n * L * h * 4 if ws is None else ws, None)
    elif entry == "ps_self_attention_forward":
        rc = f(n, L, h, d, p[0], s, p[1], 0, None)
    elif entry == "ps_self_attention_forward_stats":
        rc = f(n, L, h, d, p[0], s, p[1], p[2], None)
    else:
        rc = f(n, L, h, d, p[0], p[1], p[2], p[3], s, p[4], None)
    out.append([rc, _lib.lib.ps_last_error().decode()])
print(json.dumps(out))
"""


@pytest.fixture(scope="module")
def results():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-c", CHILD, json.dumps(VIT_PTRS), json.dumps(CASES)], cwd=str(ROOT),
                       env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    return dict(zip([c[0] for c in CASES], json.loads(r.stdout.strip().splitlines()[-1])))


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_refuses_before_enqueuing(results, case):
    rc, err = results[case[0]]
    assert rc == case[-1], err


def test_a_valid_call_reaches_the_device(results):
    """The same child with valid arguments gets past the checks: without a GPU it fails in CUDA (2), not in them."""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    cases = [("ok-" + e, e, VIT_OK if "vit" in e else SA_OK, 0.125, {}, None, 2) for e in VIT_PTRS]
    r = subprocess.run([sys.executable, "-c", CHILD, json.dumps(VIT_PTRS), json.dumps(cases)], cwd=str(ROOT),
                       env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    for case, (rc, err) in zip(cases, json.loads(r.stdout.strip().splitlines()[-1])):
        assert rc == 2, (case[0], rc, err)
