"""Float64 restatement of the two dense attention kernels, with a per-entry error bar for every output.

    out = softmax(q k^T * scale) v,   d_qkv = its gradient for the upstream gradient d_out

- the flash-style ViT attention (csrc/vit_attention.cu): any L, 64-dim heads; saves lse = ln sum_j exp(s_ij scale);
- the 256-token self-attention (csrc/self_attention_tc.cu): L = 256, 128-dim heads; saves stats = (max_j s_ij *
  scale * log2 e, 1 / sum_j exp2(s_ij scale log2 e - that max)) per row.

The restatement takes q, k, v and d_out rounded to TF32 exactly as the kernels round them on the way into shared
memory (cvt.rna.tf32: nearest, ties away from zero) and is otherwise exact float64 mathematics.  The TF32 rounding
of the inputs is inherent to running the products on the tensor cores and is not a defect: it is the same for the
kernel and the restatement, so it does not enter the bars.  (The existing whole-tensor tests compare against the
unrounded inputs and keep that error in their bars.)

The bars come from an error model of the kernel's arithmetic, one term per rounding it performs:

- each TF32 rounding of an intermediate (P before P V, P once more in the self-attention backward, dS before
  dQ / dK) costs U_TF32 relative to the rounded value;
- each float32 accumulation over n terms costs EPS_F32 * sqrt(n) * sum |terms|;
- a logit carries the accumulation error of q . k, and exp2f / the fp32 scaling add a few EPS_F32 more (P_ELEM).

Magnitudes are centred where the mathematics allows: a relative error d_j on the probabilities moves the output
by sum_j P_ij d_j (v_jc - O_ic) (the normalisation is over the same perturbed values), which is bounded through
Cauchy-Schwarz by sqrt(sum_j P_ij d_j^2) * sqrt(sum_j P_ij (v_jc - O_ic)^2); the probability error of dS
multiplies P_ij |dP_ij - D_i|.  Every bar carries the factor SLACK, so that a correct kernel sits at or below
1 / SLACK of the first-order bound and the terms neglected here (second order, the tensor core's accumulation
order) have room.

Everything runs in float64 on the inputs' device, in blocks of query rows, so that L = 16384 fits.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch

U_TF32 = 2.0 ** -11          # unit roundoff of a TF32 rounding (10 explicit mantissa bits)
EPS_F32 = 2.0 ** -24         # unit roundoff of a float32 operation
P_ELEM = 4                   # EPS_F32 units of a probability's elementwise math: s * scale log2 e - max, exp2f
SLACK = 2.0                  # every bar is SLACK x the first-order bound
LOG2E = 1.4426950408889634
VIT_TILE = 64                # keys per online soft-max step of the ViT forward (one alpha rescale each)
BLOCK_ELEMS = 1 << 26        # float64 elements of one [images x heads, rows, L] block


def _tf32(t):
    # cvt.rna.tf32.f32: nearest TF32, ties away from zero (sign-magnitude, so +0x1000 on the bits)
    return ((t.contiguous().view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)


def split_heads(x, heads):
    """[n, L, heads * d] -> [n * heads, L, d]."""
    n, L, inner = x.shape
    return x.reshape(n, L, heads, inner // heads).transpose(1, 2).reshape(n * heads, L, inner // heads)


def merge_heads(x, n):
    """[n * heads, L, d] -> [n, L, heads * d]."""
    B, L, d = x.shape
    return x.reshape(n, B // n, L, d).transpose(1, 2).reshape(n, L, -1)


@dataclass
class Restatement:
    kind: str                  # "vit" or "sa"
    heads: int
    out: torch.Tensor          # [n, L, H d]
    lse: torch.Tensor          # [n, H, L]       (ViT)
    stats: torch.Tensor        # [n, H, L, 2]    (self-attention)
    d_qkv: torch.Tensor        # [n, L, 3 H d]
    bar_out: torch.Tensor
    bar_lse: torch.Tensor
    bar_stats: torch.Tensor
    bar_d_qkv: torch.Tensor


def restate(kind, qkv, d_out, heads, scale):
    """Float64 outputs and bars of the `kind` ("vit" / "sa") kernel for float32 qkv [n, L, 3 H d], d_out [n, L, H d]."""
    assert kind in ("vit", "sa")
    n, L, _ = qkv.shape
    u, e = U_TF32, EPS_F32
    q, k, v = (split_heads(_tf32(t).double(), heads) for t in qkv.chunk(3, dim=-1))
    do = split_heads(_tf32(d_out).double(), heads)
    B, _, d = q.shape
    aq, ak, av, ado = q.abs(), k.abs(), v.abs(), do.abs()
    rd, rL = math.sqrt(d), math.sqrt(L)
    n_tiles = -(-L // VIT_TILE)
    vc = v.mean(1, keepdim=True)                                   # centre of the values: stable variances
    out = torch.empty_like(q); bar_out = torch.empty_like(q)
    dq = torch.empty_like(q); bar_dq = torch.empty_like(q)
    dk = torch.zeros_like(k); bar_dk = torch.zeros_like(k)
    dv = torch.zeros_like(v); bar_dv = torch.zeros_like(v)
    lse = q.new_empty(B, L); bar_lse = q.new_empty(B, L)
    stats = q.new_empty(B, L, 2); bar_stats = q.new_empty(B, L, 2)
    rows = max(1, min(L, BLOCK_ELEMS // (B * L)))
    for i0 in range(0, L, rows):
        sl = slice(i0, min(L, i0 + rows))
        s = q[:, sl] @ k.transpose(1, 2)                           # [B, r, L] raw logits
        m = s.amax(-1, keepdim=True)
        ex = torch.exp((s - m) * scale)
        Z = ex.sum(-1, keepdim=True)
        P = ex / Z
        O = P @ v
        # relative error of one probability before any TF32 rounding: the logit's accumulation error, the fp32
        # scaling and max subtraction, exp2f
        d_s = e * rd * (aq[:, sl] @ ak.transpose(1, 2))
        delta = abs(scale) * (d_s + P_ELEM * e * (s.abs() + m.abs())) + P_ELEM * e
        del ex, d_s
        # output: P rounded to TF32 before P V (centred), the P V accumulation, the normalisation (and for the
        # ViT, one alpha rescale of O and of the row sum per key tile)
        e_fwd = u + delta
        spread = ((P @ (v - vc).square()) - (O - vc).square()).clamp_min(0).sqrt()
        n_norm = 2 + (2 * n_tiles if kind == "vit" else 0)
        b_out = ((P * e_fwd.square()).sum(-1, keepdim=True).sqrt() * spread
                 + e * rL * (P @ av) + e * n_norm * O.abs())
        # row statistics
        e_sum = (P * e_fwd).sum(-1) + e * (rL + n_norm)           # relative error of the kernel's row sum
        mlog = m[..., 0] * scale                                   # max logit, natural units
        lse_b = mlog + torch.log(Z[..., 0])
        if kind == "vit":
            b_lse = e_sum + P_ELEM * e * (lse_b.abs() + mlog.abs())
            e_norm = b_lse + 2 * e * lse_b.abs()                   # lse * log2 e in fp32 in the backward
            lse[:, sl], bar_lse[:, sl] = lse_b, b_lse
        else:
            b_mb = LOG2E * (abs(scale) * e * rd * (aq[:, sl] @ ak.transpose(1, 2)).amax(-1)
                            + P_ELEM * e * mlog.abs())
            inv = 1.0 / Z[..., 0]
            b_inv = inv * (math.log(2.0) * b_mb + e_sum)
            stats[:, sl, 0], stats[:, sl, 1] = mlog * LOG2E, inv
            bar_stats[:, sl, 0], bar_stats[:, sl, 1] = b_mb, b_inv
            e_norm = b_inv / inv + e + u                           # Pn = tf32(p) * inv
        out[:, sl], bar_out[:, sl] = O, b_out
        # backward
        dP = do[:, sl] @ v.transpose(1, 2)
        D = (do[:, sl] * O).sum(-1, keepdim=True)
        dS = P * (dP - D) * scale
        e_ds = delta + e_norm[..., None]                           # the P dS is formed from
        e_dv = e_ds + u                                            # P rounded to TF32 before dV = P^T dO
        d_term = (e * rd * (ado[:, sl] * O.abs()).sum(-1, keepdim=True)           # D's accumulation
                  + (ado[:, sl] * b_out).sum(-1, keepdim=True))                   # D from the kernel's O
        b_ds = (abs(scale) * P * (e_ds * (dP - D).abs() + e * rd * (ado[:, sl] @ av.transpose(1, 2)) + d_term)
                + 3 * e * dS.abs())
        del dP, delta
        a_ds = dS.abs() * (u + e * rL)                             # dS rounded to TF32, dQ / dK accumulation
        dq[:, sl] = dS @ k
        bar_dq[:, sl] = (b_ds + a_ds) @ ak
        dk += dS.transpose(1, 2) @ q[:, sl]
        bar_dk += (b_ds + a_ds).transpose(1, 2) @ aq[:, sl]
        dv += P.transpose(1, 2) @ do[:, sl]
        bar_dv += (P * (e_dv + e * rL)).transpose(1, 2) @ ado[:, sl]
        del s, P, dS, b_ds, a_ds, e_fwd, e_ds, e_dv
    c = SLACK
    return Restatement(
        kind, heads,
        out=merge_heads(out, n), lse=lse.reshape(n, heads, L), stats=stats.reshape(n, heads, L, 2),
        d_qkv=torch.cat([merge_heads(t, n) for t in (dq, dk, dv)], -1),
        bar_out=c * merge_heads(bar_out, n), bar_lse=c * bar_lse.reshape(n, heads, L),
        bar_stats=c * bar_stats.reshape(n, heads, L, 2),
        bar_d_qkv=c * torch.cat([merge_heads(t, n) for t in (bar_dq, bar_dk, bar_dv)], -1))


# ----------------------------------------------------------------------------------------------- locating a failure

def _where(kind, tensor, idx, shape, heads):
    """The kernel coordinates of entry `idx` (a tuple into `shape`) of `tensor`."""
    if tensor in ("lse", "stats"):
        img, head, tok = idx[:3]
        ch = ("max", "inv")[idx[3]] if tensor == "stats" else None
        part = tensor
    else:
        img, tok, col = idx
        d = shape[-1] // heads // (3 if tensor == "d_qkv" else 1)
        part = "out" if tensor == "out" else "dq dk dv".split()[col // (heads * d)]
        head, ch = (col % (heads * d)) // d, col % d
    tile, wg = tok // 128, (tok % 128) // 64
    if kind == "vit":
        kern = {"out": "fwd", "lse": "fwd", "dq": "bwd_dq", "dk": "bwd_dkdv", "dv": "bwd_dkdv"}[part]
        cta = f"k_vit_attn_{kern} tile {tile}"
    elif part in ("out", "stats"):
        cta = f"forward half {tile}"
    elif part == "dq":
        cta = f"backward role 0 (dQ) half {tile}"
    else:
        cta = f"backward role 1 (dK, dV) half {tile}"
    return f"{part} image {img} head {head} token {tok} channel {ch}: CTA {cta} warpgroup {wg}"


def ratio(got, ref, bar):
    """|got - ref| / bar per entry (inf where the kernel's value is not finite)."""
    r = (got.double() - ref).abs() / bar
    return torch.where(torch.isfinite(got), r, torch.full_like(r, math.inf))


def check(kind, name, got, ref, bar, heads, limit=1.0):
    """Asserts every entry of `got` is within `limit` x its bar; the message locates the worst one."""
    r = ratio(got, ref, bar)
    worst = float(r.max())
    if worst > limit:
        idx = tuple(int(i) for i in torch.unravel_index(torch.argmax(r.nan_to_num(math.inf)), r.shape))
        raise AssertionError(
            f"{_where(kind, name, idx, tuple(r.shape), heads)}: got {float(got[idx]):.9g}, float64 "
            f"{float(ref[idx]):.9g}, error / bar = {worst:.3g} ({int((r > limit).sum())} entries over)")
    return worst


def worst_ratios(kind, res, out, side, d_qkv):
    """Worst error / bar per tensor: out, lse or stats (`side`), dq, dk, dv."""
    got = {"out": ratio(out, res.out, res.bar_out)}
    if kind == "vit":
        got["lse"] = ratio(side, res.lse, res.bar_lse)
    else:
        got["stats"] = ratio(side, res.stats, res.bar_stats)
    for nm, a, b, c in zip(("dq", "dk", "dv"), d_qkv.chunk(3, -1), res.d_qkv.chunk(3, -1), res.bar_d_qkv.chunk(3, -1)):
        got[nm] = ratio(a, b, c)
    return {nm: float(r.max()) for nm, r in got.items()}


def check_all(kind, res, out, side, d_qkv):
    """`check` on every output of one run; returns the worst ratio per tensor."""
    w = {"out": check(kind, "out", out, res.out, res.bar_out, res.heads)}
    if kind == "vit":
        w["lse"] = check(kind, "lse", side, res.lse, res.bar_lse, res.heads)
    else:
        w["stats"] = check(kind, "stats", side, res.stats, res.bar_stats, res.heads)
    r = ratio(d_qkv, res.d_qkv, res.bar_d_qkv)
    check(kind, "d_qkv", d_qkv, res.d_qkv, res.bar_d_qkv, res.heads)
    for nm, part in zip(("dq", "dk", "dv"), r.chunk(3, -1)):
        w[nm] = float(part.max())
    return w


# ------------------------------------------------------------------------------------------------- input families

# name -> scale (None: d ** -0.5, the modules' own)
FAMILIES = {
    "randn": None,
    "v_offset3": None,         # V = 0.1 randn + 3 c, c a +-1 vector shared by every token
    "v_offset10": None,        # V = 0.1 randn + 10 c
    "q_offset": None,          # Q with a common offset of 3 spreads: logits vary strongly by key
    "k_offset": None,          # K with a common offset of 3 spreads: a per-row shift of the logits
    "near_uniform": None,      # q, k of spread 0.05
    "peaked": None,            # q, k of spread 3
    "one_hot": 1.0,            # query i matches key perm[i] overwhelmingly
    "do_offset": None,         # d_out with a common offset of 3 spreads
    "scale_0.125": 0.125,
    "scale_128^-0.5": 128 ** -0.5,
    "scale_1": 1.0,
    "scale_1e-3": 1e-3,
}


def make_inputs(family, n, L, heads, d, seed):
    """float32 (qkv [n, L, 3 H d], d_out [n, L, H d], scale) of one input family, on the CPU."""
    g = torch.Generator().manual_seed(seed)
    shape = (n, L, heads * d)
    q, k, v, do = (torch.randn(shape, generator=g) for _ in range(4))
    common = lambda: torch.randint(0, 2, (1, 1, heads * d), generator=g).float() * 2 - 1
    if family.startswith("v_offset"):
        v = 0.1 * v + float(family[len("v_offset"):]) * common()
    elif family == "q_offset":
        q = q + 3 * common()
    elif family == "k_offset":
        k = k + 3 * common()
    elif family == "near_uniform":
        q, k = 0.05 * q, 0.05 * k
    elif family == "peaked":
        q, k = 3 * q, 3 * k
    elif family == "do_offset":
        do = do + 3 * common()
    elif family == "one_hot":
        basis = torch.randn(L, d, generator=g)
        basis = basis / basis.norm(dim=-1, keepdim=True) * (40.0 if d == 128 else 60.0)
        k = basis[None, :, None, :].expand(n, L, heads, d)
        q = torch.stack([torch.stack([basis[torch.randperm(L, generator=g)] for _ in range(heads)], 1)
                         for _ in range(n)])
        q, k = q.reshape(shape), k.reshape(shape)
    scale = FAMILIES[family]
    return torch.cat([q, k, v], -1).contiguous(), do.contiguous(), d ** -0.5 if scale is None else scale
