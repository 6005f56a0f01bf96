"""CPU tests of the host surface of the fixed-order epipolar attention backward
(include/pixelsplat_b200.h ps_epipolar_attention_backward_workspace_bytes / _deterministic): both symbols are
exported and bound, the workspace query needs no device and equals the header's formula, and both entry points
reject a bad descriptor, NULL pointers and a short workspace before anything touches a device."""
import ctypes

import pytest

align = lambda x: (x + 255) // 256 * 256
FAKE = ctypes.c_void_p(0x1000)          # never dereferenced: every call below is refused before any launch


def _desc(b, v, h, w, S, heads=4, pe_dim=20, channels=128):
    from pixelsplat_b200 import _lib
    return _lib.EpipolarDesc(b, v, h, w, S, channels, heads, pe_dim)


def _formula(b, v, h, w, S):
    T = b * v * h * w * (v - 1) * S
    cells = b * v * (h + 1) * (w + 1)
    return (align(512 * T) + align(16 * T) + 4 * align(4 * T) + align(1024 * -(-T // 4096))
            + align(4 * (cells + 1)) + align(2048 * cells))


def _inputs():
    from pixelsplat_b200 import _lib
    return _lib.EpipolarInputs(*([FAKE.value] * 7))


def _bytes(d):
    from pixelsplat_b200 import _lib
    out = ctypes.c_size_t()
    rc = _lib.lib.ps_epipolar_attention_backward_workspace_bytes(ctypes.byref(d), ctypes.byref(out))
    return rc, out.value


def test_symbols_are_exported_and_bound():
    from pixelsplat_b200 import _lib
    for name in ("ps_epipolar_attention_backward_workspace_bytes", "ps_epipolar_attention_backward_deterministic"):
        assert name in _lib.EXPORTS
        fn = getattr(_lib.lib, name)
        assert fn.restype is ctypes.c_int and fn.argtypes
    assert len(_lib.lib.ps_epipolar_attention_backward_deterministic.argtypes) == 14


@pytest.mark.parametrize("shape", [(2, 3, 6, 10, 7), (7, 2, 64, 64, 32)])
def test_workspace_equals_the_header_formula(shape):
    """A small shape and configs[2] at batch 7 (64 x 64 rays, S = 32, two views): about 1.1 GB there."""
    from pixelsplat_b200 import _lib
    d = _desc(*shape)
    want = _formula(*shape)
    assert _bytes(d) == (0, want)
    assert _lib.epipolar_backward_workspace_bytes(d) == want
    if shape[0] == 7:
        assert 1.0e9 < want < 1.3e9


BAD = [dict(b=0), dict(v=1), dict(h=0), dict(w=0), dict(channels=64), dict(heads=0), dict(heads=5), dict(S=0),
       dict(S=33), dict(pe_dim=3), dict(pe_dim=34), dict(heads=4, pe_dim=32), dict(v=34)]


@pytest.mark.parametrize("bad", BAD, ids=[",".join(f"{k}={v}" for k, v in b.items()) for b in BAD])
def test_rejects_what_the_descriptor_check_rejects(bad):
    """The same return code as the forward's descriptor check, for the query and the deterministic backward."""
    from pixelsplat_b200 import _lib
    args = dict(b=1, v=2, h=4, w=4, S=8, heads=2, pe_dim=8, channels=128)
    args.update(bad)
    d = _desc(**args)
    ref = _lib.lib.ps_epipolar_attention_forward(ctypes.byref(d), ctypes.byref(_inputs()), FAKE, FAKE, FAKE, FAKE, None)
    assert ref != 0
    assert _bytes(d)[0] == ref
    rc = _lib.lib.ps_epipolar_attention_backward_deterministic(
        ctypes.byref(d), ctypes.byref(_inputs()), *([FAKE] * 9), FAKE, 1 << 40, None)
    assert rc == ref
    with pytest.raises((ValueError, _lib.NativeError)):
        _lib.epipolar_backward_workspace_bytes(d)


def test_query_rejects_null_out():
    from pixelsplat_b200 import _lib
    assert _lib.lib.ps_epipolar_attention_backward_workspace_bytes(ctypes.byref(_desc(1, 2, 4, 4, 8)), None) == 1


# argument positions of ps_epipolar_attention_backward_deterministic after (desc, inputs)
PTRS = ["lse", "dz", "de", "dmass", "d_row", "dq_feat", "dq_pe", "dbias", "dfeatures", "workspace"]
REQUIRED = ["lse", "dz", "de", "d_row", "dq_feat", "dq_pe", "dfeatures", "workspace"]
INPUTS = ["features", "segments", "valid", "rel_disparity", "q_feat", "q_pe"]


@pytest.mark.parametrize("null", REQUIRED + ["in." + n for n in INPUTS] + ["desc", "inputs"])
def test_rejects_null_pointers_before_touching_a_device(null):
    from pixelsplat_b200 import _lib
    d = _desc(1, 2, 4, 4, 8, heads=2, pe_dim=8)
    need = _lib.epipolar_backward_workspace_bytes(d)
    inp = _inputs()
    if null.startswith("in."):
        setattr(inp, null[3:], None)
    ptrs = [None if p == null else FAKE for p in PTRS]
    rc = _lib.lib.ps_epipolar_attention_backward_deterministic(
        None if null == "desc" else ctypes.byref(d), None if null == "inputs" else ctypes.byref(inp), *ptrs, need,
        None)
    assert rc == 1, _lib.lib.ps_last_error()


def test_rejects_a_one_byte_short_workspace():
    from pixelsplat_b200 import _lib
    d = _desc(2, 3, 6, 10, 7, heads=3, pe_dim=20)
    need = _lib.epipolar_backward_workspace_bytes(d)
    rc = _lib.lib.ps_epipolar_attention_backward_deterministic(ctypes.byref(d), ctypes.byref(_inputs()),
                                                               *([FAKE] * 10), need - 1, None)
    assert rc == 1
    assert b"workspace" in _lib.lib.ps_last_error()
