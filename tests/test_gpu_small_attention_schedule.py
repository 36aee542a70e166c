"""The CUDA-core attention kernels of the conditioning path at the edges of their launch policies, against float64.

`small_attention_kernel` (`ladi_attention_small`: the CLIP text and vision towers and the inversion adapter's full encoder layers) splits
the query rows of one (head, image) over `chunks` blocks of `rows_per_block` rows, warp w taking rows w, w + 8, ...; a causal block
loads only the keys its last row sees.  `cls_attention_kernel` (`ladi_cls_attention`: the adapter's last layer) strides 128 threads
over tokens for the scores and over head columns for P.V.  `ladi_attention_small_plan` / `ladi_cls_attention_plan` report what the
launches run; they share the validation-and-policy function with the launches and need no device.  Every GPU case first asserts,
through the query at 132 SMs, the plan it means to exercise (on a 132-SM H100 SXM that is also the plan that runs).  It then goes
through the census checkers (`check_attention_small`, `check_cls` in tests/kernel_check.py): every input pitch gap and the gaps between images are NaN, the
output is NaN over its full pitch, between images and in a tail, afterwards exactly the rows and columns the call owns are finite, a
second run is bit-identical, and every query row of every image is within the float64 bound (attn_expect with P in fp32).

Score distributions: "randn" (q, k ~ N(0, 2), the census's), "unit" (N(0, 1)), "late" (the scores grow along the keys, so a causal
row's maximum sits on its diagonal and the last keys dominate), "large" (scores near +-80 / scale before the maximum is subtracted).

The CPU tests pin the plan tables and every placement rule through the queries, and show the checkers have teeth: a float32 emulation
of each kernel's block and warp split, driven by the queried plan, passes, and four simulated faults are rejected."""
import time
import zlib

import numpy as np
import pytest
import torch

from kernel_check import (NAN, SMS, Replay, addr, attn_expect, attn_ref, check_attention_small, check_cls, ladi_lib, launches, override,
                          plan_query, ratio, small_attn_expect, sms)

OPTIN = 48 * 1024


# ================================================================================================================ queries
SA_ORDER = ("q", "k", "v", "out", "B", "heads", "nq", "nkv", "hd", "qp", "kp", "vp", "op", "qbs", "kbs", "vbs", "obs", "scale", "causal")
PLAN_FIELDS = ("chunks", "rows_per_block", "smem_bytes", "smem_optin")


def sa_desc(B, heads, nq, nkv, hd, causal=0, **kw):
    """ladi_attention_small's arguments in the glue census's field names: dense [B, n, heads*hd] operands on fake 256-byte aligned
    addresses; kw overrides by name, *_off adds a byte offset to a pointer."""
    Cw = heads * hd
    return override(dict(q=addr(1), k=addr(2), v=addr(3), out=addr(4), B=B, heads=heads, nq=nq, nkv=nkv, hd=hd, qp=Cw, kp=Cw, vp=Cw,
                          op=Cw, qbs=nq * Cw, kbs=nkv * Cw, vbs=nkv * Cw, obs=nq * Cw, scale=hd ** -0.5, causal=causal), kw)


def sa_query(d, sms=SMS):
    """-> (plan dict, "") or (None, error message)."""
    return plan_query("ladi_attention_small_plan", ladi_lib().SmallAttnPlan, [d[k] for k in SA_ORDER] + [sms], PLAN_FIELDS)


CLS_ORDER = ("q", "qp", "kv", "kvp", "batch", "tokens", "heads", "hd", "scale", "out", "op")


def cls_desc(B, T, heads, hd, **kw):
    """ladi_cls_attention's arguments in the workload census's field names (dense, fake addresses), overridden like sa_desc."""
    Cw = heads * hd
    return override(dict(q=addr(1), qp=Cw, kv=addr(2), kvp=2 * Cw, batch=B, tokens=T, heads=heads, hd=hd, scale=hd ** -0.5, out=addr(3),
                          op=Cw), kw)


def cls_query(d, sms=SMS):
    return plan_query("ladi_cls_attention_plan", ladi_lib().SmallAttnPlan, [d[k] for k in CLS_ORDER] + [sms], PLAN_FIELDS)


def sa_smem(hd, nkv):
    """small_attention_kernel's dynamic shared memory: K (odd word stride) and V of one head, 8 warps' P rows (keys padded to 32) and Q."""
    return nkv * (hd + 1) * 4 + 8 * (-(-nkv // 32) * 32) * 4 + 8 * hd * 4


# ================================================================================================================ CPU: plan tables
# (B, heads, nq, nkv, hd, causal) -> (chunks, rows_per_block, smem_bytes, smem_optin) at 132 and at 114 SMs:
# chunks = ceil(2 SMs / (B heads)), rows_per_block = max(8, ceil(nq / chunks)), then chunks = ceil(nq / rows_per_block).
SA_TABLE = [
    ("vision tower / adapter encoder layer", (8, 16, 257, 257, 80, 0), (3, 86, 95044, 1), (2, 129, 95044, 1)),
    ("text tower", (8, 16, 77, 77, 64, 1), (3, 26, 25140, 0), (2, 39, 25140, 0)),
    ("one chunk, 33 rows per warp", (17, 16, 257, 257, 64, 0), (1, 257, 78084, 1), (1, 257, 78084, 1)),
    ("rows_per_block floor", (1, 1, 100, 100, 64, 0), (13, 8, 32144, 0), (13, 8, 32144, 0)),
    ("rows_per_block 13", (3, 4, 280, 280, 64, 0), (22, 13, 84064, 1), (19, 15, 84064, 1)),
    ("last block 1 row", (1, 2, 257, 257, 64, 0), (33, 8, 78084, 1), (33, 8, 78084, 1)),
    ("nq 1", (2, 4, 1, 50, 64, 0), (1, 8, 17096, 0), (1, 8, 17096, 0)),
    ("causal 77, 2 chunks", (9, 16, 77, 77, 64, 1), (2, 39, 25140, 0), (2, 39, 25140, 0)),
    ("causal 77, 10 chunks", (1, 2, 77, 77, 64, 1), (10, 8, 25140, 0), (10, 8, 25140, 0)),
    ("causal 257, 2 chunks", (9, 16, 257, 257, 64, 1), (2, 129, 78084, 1), (2, 129, 78084, 1)),
    ("causal 1000, 125 chunks", (1, 2, 1000, 1000, 40, 1), (125, 8, 198048, 1), (112, 9, 198048, 1)),
    ("causal 1000, 3 chunks", (1, 100, 1000, 1000, 40, 1), (3, 334, 198048, 1), (3, 334, 198048, 1)),
    ("causal 1000, 2 chunks", (2, 70, 1000, 1000, 40, 1), (2, 500, 198048, 1), (2, 500, 198048, 1)),
    ("head width 128, largest nkv", (1, 2, 100, 365, 128, 0), (13, 8, 204724, 1), (13, 8, 204724, 1)),
    ("1024 keys at head width 40", (1, 4, 1, 1024, 40, 0), (1, 8, 201984, 1), (1, 8, 201984, 1)),
    ("1024 keys at head width 8", (2, 3, 64, 1024, 8, 0), (8, 8, 69888, 1), (8, 8, 69888, 1)),
    ("cross attention, 5 keys", (2, 2, 300, 5, 64, 0), (38, 8, 4372, 0), (38, 8, 4372, 0)),
]


@pytest.mark.parametrize("name,shape,at132,at114", SA_TABLE, ids=[t[0] for t in SA_TABLE])
def test_attention_small_plan_table(name, shape, at132, at114):
    *dims, causal = shape
    for sms, want in ((132, at132), (114, at114)):
        p, err = sa_query(sa_desc(*dims, causal=causal), sms)
        assert p is not None, err
        assert tuple(p.values()) == want, (sms, p)
        assert p["smem_bytes"] == sa_smem(dims[4], dims[3])


def test_attention_small_shared_memory_limit():
    """200 KB: at head width 128 the last accepted key count is 365; 1024 keys fit at head width 40 (201984 bytes) and not at 48."""
    assert sa_query(sa_desc(1, 2, 100, 365, 128))[0]["smem_bytes"] == 204724
    for hd, nkv in ((128, 366), (48, 1024), (64, 694)):
        p, err = sa_query(sa_desc(1, 2, 100, nkv, hd))
        assert p is None and "do not fit shared memory" in err, (hd, nkv)
    assert sa_query(sa_desc(1, 2, 100, 693, 64))[0] is not None
    assert sa_query(sa_desc(1, 2, 100, 1024, 40))[0]["smem_bytes"] == 201984
    p, err = sa_query(sa_desc(1, 2, 100, 1025, 8))
    assert p is None and "nkv <= 1024" in err


def test_attention_small_plan_covers_every_row():
    """For every (B heads, nq) the blocks tile the rows exactly: rows_per_block >= 8, chunks blocks, the last one non-empty."""
    for bh in (1, 2, 3, 7, 12, 16, 44, 66, 128, 131, 132, 133, 263, 264, 265, 1000):
        for nq in (1, 7, 8, 9, 77, 100, 257, 280, 1000):
            for sms in (114, 132):
                p, _ = sa_query(sa_desc(1, bh, nq, 8, 8), sms)
                assert p["rows_per_block"] >= 8 and (p["chunks"] - 1) * p["rows_per_block"] < nq <= p["chunks"] * p["rows_per_block"]


def test_cls_plan_and_token_limit():
    """One block per (head, image); the query and the token probabilities in fp32 plus the 16 bytes of static reduction slots within
    48 KB: 12204 tokens at head width 80, not 12205."""
    p, err = cls_query(cls_desc(8, 257, 16, 80))
    assert p == dict(chunks=1, rows_per_block=1, smem_bytes=(80 + 257) * 4, smem_optin=0), err
    p, err = cls_query(cls_desc(1, 12204, 1, 80))
    assert p is not None and p["smem_bytes"] + 16 == OPTIN, err
    p, err = cls_query(cls_desc(1, 12205, 1, 80))
    assert p is None and "too many tokens" in err


# ================================================================================================================ CPU: placement rules
SA_REJECT = [  # (name, overrides, word the message must contain)
    ("k 8-byte aligned", dict(k_off=8), "k "),
    ("v 4-byte aligned", dict(v_off=4), "v "),
    ("q 2-byte aligned", dict(q_off=2), "q "),
    ("out 2-byte aligned", dict(out_off=2), "out "),
    ("q_pitch below the width", dict(qp=120), "q_pitch"),
    ("k_pitch below the width", dict(kp=120), "k_pitch"),
    ("v_pitch below the width", dict(vp=64), "v_pitch"),
    ("out_pitch below the width", dict(op=120), "out_pitch"),
    ("out images overlap", dict(obs=10 * 128 - 8), "out_batch_stride"),
    ("pitch not a multiple of 8", dict(kp=132), "multiples of 8"),
    ("batch stride not a multiple of 8", dict(vbs=20 * 128 + 4), "multiples of 8"),
    ("causal with nq != nkv", dict(causal=1), "causal"),
    ("head width not a multiple of 8", dict(hd=12, heads=10, qp=120, kp=120, vp=120, op=120), "head_dim"),
    ("null q", dict(q=None), "null"),
]


@pytest.mark.parametrize("name,kw,word", SA_REJECT, ids=[r[0] for r in SA_REJECT])
def test_attention_small_placement_rejected(name, kw, word):
    p, err = sa_query(override(sa_desc(2, 2, 10, 20, 64), kw))
    assert p is None, f"{name}: accepted"
    assert word in err, err


SA_ACCEPT = [
    ("q and out 4-byte aligned", dict(q_off=4, out_off=12)),
    ("k and v 16-byte aligned", dict(k_off=16, v_off=48)),
    ("fused QKV", dict(k=addr(1, 256), v=addr(1, 512), qp=384, kp=384, vp=384, qbs=10 * 384 + 8, kbs=10 * 384 + 8, vbs=10 * 384 + 8)),
    ("input images overlap (batch stride 0)", dict(kbs=0, vbs=0)),
    ("out images with gaps", dict(obs=10 * 136 + 8, op=136)),
    ("one image: out_batch_stride unused", dict(B=1, obs=0)),
]


@pytest.mark.parametrize("name,kw", SA_ACCEPT, ids=[r[0] for r in SA_ACCEPT])
def test_attention_small_placement_accepted(name, kw):
    p, err = sa_query(override(sa_desc(2, 2, 10, 10 if "fused" in name else 20, 64), kw))
    assert p is not None, err


CLS_REJECT = [
    ("kv 2-byte aligned", dict(kv_off=2), "kv "),
    ("kv_pitch below 2 heads hd", dict(kvp=2 * 160 - 2), "kv_pitch"),
    ("kv_pitch odd", dict(kvp=2 * 160 + 1), "kv_pitch"),
    ("q_pitch below heads hd", dict(qp=158), "q_pitch"),
    ("out_pitch below heads hd", dict(op=150), "out_pitch"),
    ("odd head width", dict(hd=81), "bad arguments"),
    ("null kv", dict(kv=None), "bad arguments"),
]


@pytest.mark.parametrize("name,kw,word", CLS_REJECT, ids=[r[0] for r in CLS_REJECT])
def test_cls_placement_rejected(name, kw, word):
    p, err = cls_query(override(cls_desc(2, 30, 2, 80), kw))
    assert p is None, f"{name}: accepted"
    assert word in err, err


def test_cls_placement_accepted():
    """q0 and out are read and written as scalars (2-byte aligned is enough); kv 4-byte aligned; pitches above the widths."""
    for kw in (dict(q_off=2, out_off=6), dict(kv_off=4), dict(qp=168, kvp=330, op=162)):
        p, err = cls_query(cls_desc(2, 30, 2, 80, **kw))
        assert p is not None, (kw, err)


def test_production_placements_accepted():
    """The placements of the production callers: clip.py / adapter.py's encoder layer (q, k, v as column slices of one fused QKV GEMM
    output, a fresh dense output) and csrc/engine.cu's (the same on workspace blocks of 256 bytes), and the adapter's CLS attention."""
    for B, heads, T, hd, causal in ((8, 16, 77, 64, 1), (8, 16, 257, 80, 0)):
        Cw = heads * hd
        qkv = addr(1)
        d = sa_desc(B, heads, T, T, hd, causal=causal, q=qkv, k=qkv + 2 * Cw, v=qkv + 4 * Cw, qp=3 * Cw, kp=3 * Cw, vp=3 * Cw,
                    qbs=T * 3 * Cw, kbs=T * 3 * Cw, vbs=T * 3 * Cw)
        assert sa_query(d)[0] is not None
    assert cls_query(cls_desc(8, 257, 16, 80))[0] is not None


def test_ops_plan_queries():
    """ops.attention_small_plan / ops.cls_attention_plan on the Python callers' views (host tensors: the queries read no memory)."""
    from ladi_vton_b200 import ops
    C_ = 1280
    qkv = torch.empty((8, 257, 3 * C_), dtype=torch.bfloat16)
    p = ops.attention_small_plan(qkv[..., :C_], qkv[..., C_:2 * C_], qkv[..., 2 * C_:], 16, 80 ** -0.5, sms=132)
    assert (p.chunks, p.rows_per_block, p.smem_bytes, p.smem_optin) == (3, 86, 95044, 1)
    with pytest.raises(RuntimeError, match="v_pitch"):
        ops.attention_small_plan(qkv[..., :C_], qkv[..., C_:2 * C_], torch.empty((8, 257, 640), dtype=torch.bfloat16), 16, 0.1, sms=132)
    kv = torch.empty((8, 257, 2 * C_), dtype=torch.bfloat16)
    p = ops.cls_attention_plan(torch.empty((8, C_), dtype=torch.bfloat16), kv, 16, 80, 80 ** -0.5)
    assert (p.chunks, p.rows_per_block, p.smem_bytes, p.smem_optin) == (1, 1, (80 + 257) * 4, 0)
    with pytest.raises(RuntimeError, match="kv_pitch"):
        ops.cls_attention_plan(torch.empty((8, C_), dtype=torch.bfloat16), torch.empty((8, 257, C_), dtype=torch.bfloat16), 16, 80, 80 ** -0.5)


# ================================================================================================================ CPU: the checkers have teeth
def _f32(t):
    return t.float().numpy()


def emulate_small(q, k, v, heads, scale, causal, rpb, fault=None):
    """fp32 emulation of small_attention_kernel for one image: blocks of rpb rows, each loading min(nkv, r1) keys when causal; per row
    Q pre-scaled by scale log2 e, four partial dot-product sums, exp2 against the row maximum, P.V over the keys in order.  The faults:
    "short" -- a causal block loads one key fewer (the missing key reads as zero); "pair1" -- the second bf16 pair of a lane (columns
    64 and up) is dropped; "last_row" -- the last block skips its final row (the output there stays zero)."""
    nq, Cw = q.shape
    nkv, hd = k.shape[0], Cw // heads
    qf, kf, vf = _f32(q), _f32(k), _f32(v)
    sl2 = np.float32(scale) * np.float32(1.4426950408889634)
    out = np.zeros((nq, Cw), np.float32)
    nblk = -(-nq // rpb)
    for blk in range(nblk):
        r0, r1 = blk * rpb, min(nq, blk * rpb + rpb)
        loaded = min(nkv, r1) if causal else nkv
        if fault == "short" and causal:
            loaded -= 1
        rows = np.arange(r0, r1 - 1 if fault == "last_row" and blk == nblk - 1 else r1)
        visible = np.arange(nkv)[None, :] <= rows[:, None] if causal else np.ones((len(rows), nkv), bool)
        for h in range(heads):
            cs = slice(h * hd, (h + 1) * hd)
            Kh, Vh = np.zeros((nkv, hd), np.float32), np.zeros((nkv, hd), np.float32)
            Kh[:loaded], Vh[:loaded] = kf[:loaded, cs], vf[:loaded, cs]
            Q = qf[rows, cs] * sl2
            a = np.zeros((4, len(rows), nkv), np.float32)
            for i in range(0, hd, 4):
                for t in range(4):
                    a[t] += Q[:, i + t, None] * Kh[None, :, i + t]
            s = np.where(visible, (a[0] + a[1]) + (a[2] + a[3]), np.float32(-np.inf))
            p = np.exp2(s - s.max(1, keepdims=True)).astype(np.float32)
            o = np.zeros((len(rows), hd), np.float32)
            for j in range(nkv):
                o += p[:, j:j + 1] * Vh[j]
            o *= np.float32(1) / p.sum(1, keepdims=True, dtype=np.float32)
            if fault == "pair1":
                o[:, 64:] = 0
            out[rows, cs] = o
    return torch.from_numpy(out).bfloat16()


def emulate_cls(q0, kv, heads, hd, scale, fault=None):
    """fp32 emulation of cls_attention_kernel for one image; the fault "first128": only the first 128 tokens are summed."""
    Cw = heads * hd
    T = kv.shape[0] if fault != "first128" else min(128, kv.shape[0])
    qf, kf, vf = _f32(q0)[0], _f32(kv)[:T, :Cw], _f32(kv)[:T, Cw:2 * Cw]
    out = np.zeros((1, Cw), np.float32)
    for h in range(heads):
        cs = slice(h * hd, (h + 1) * hd)
        sq, K, V = qf[cs] * np.float32(scale), kf[:, cs], vf[:, cs]
        s = np.zeros(T, np.float32)
        for d in range(0, hd, 2):
            s += sq[d] * K[:, d] + sq[d + 1] * K[:, d + 1]
        e = np.exp(s - s.max()).astype(np.float32)
        acc = np.zeros(hd, np.float32)
        for t in range(T):
            acc += e[t] * V[t]
        out[0, cs] = acc * (np.float32(1) / e.sum(dtype=np.float32))
    return torch.from_numpy(out).bfloat16()


def make_qkv(g, nq, nkv, heads, hd, dist, dev="cpu"):
    """bf16 q [nq, heads hd], k / v [nkv, heads hd] with the score distribution `dist` (module docstring); scale = hd^-1/2."""
    Cw = heads * hd
    rn = lambda *s: torch.randn(s, generator=g, device=dev)  # noqa: E731
    v = rn(nkv, Cw)
    if dist in ("randn", "unit"):
        sd = 2 ** 0.5 if dist == "randn" else 1.0
        return (rn(nq, Cw) * sd).bfloat16(), (rn(nkv, Cw) * sd).bfloat16(), v.bfloat16()
    u = torch.sign(rn(1, Cw)) + 0.0  # one direction per head column
    q = u + 0.5 * rn(nq, Cw)
    if dist == "late":  # scale q.k grows by about 8 from the first key to the last
        a = 8.0 * torch.arange(nkv, device=dev, dtype=torch.float32)[:, None] / max(1, nkv - 1)
    else:  # "large": scale q.k near +80 for a random half of the keys and -80 for the rest
        a = 80.0 * torch.where(torch.rand((nkv, 1), generator=g, device=dev) < 0.5, -1.0, 1.0)
    k = a * u / hd ** 0.5 + 0.5 * rn(nkv, Cw)
    return q.bfloat16(), k.bfloat16(), v.bfloat16()


TEETH_SHAPES = [  # (B heads for the plan, heads, nq, nkv, hd, causal, dist)
    (128, 2, 77, 77, 64, 1, "late"),     # the text tower's 3 chunks of 26 rows
    (2, 2, 77, 77, 64, 1, "late"),       # 10 chunks of 8 rows
    (12, 1, 100, 100, 72, 0, "randn"),   # 4 lanes with a second pair
    (12, 1, 100, 60, 80, 0, "unit"),
    (2, 2, 33, 33, 128, 1, "late"),
    (128, 2, 77, 77, 64, 0, "large"),
    (6, 2, 40, 1024, 40, 0, "late"),
]


def _teeth_case(i, bh, heads, nq, nkv, hd, causal, dist):
    g = torch.Generator().manual_seed(100 + i)
    q, k, v = make_qkv(g, nq, nkv, heads, hd, dist)
    p, err = sa_query(sa_desc(1, bh, nq, nkv, hd, causal=causal))
    assert p is not None, err
    o, bound = small_attn_expect(q.double(), k.double(), v.double(), heads, hd ** -0.5, causal)
    return q, k, v, p["rows_per_block"], o, bound


@pytest.mark.parametrize("i", range(len(TEETH_SHAPES)))
def test_small_checker_accepts_honest_emulation(i):
    bh, heads, nq, nkv, hd, causal, dist = TEETH_SHAPES[i]
    q, k, v, rpb, o, bound = _teeth_case(i, *TEETH_SHAPES[i])
    worst = float(ratio(emulate_small(q, k, v, heads, hd ** -0.5, causal, rpb), o, bound).max())
    print(f"\n{TEETH_SHAPES[i]}: honest emulation worst err/bound {worst:.3g}")
    assert worst <= 1.0


@pytest.mark.parametrize("fault,i", [("short", 0), ("short", 1), ("short", 4), ("pair1", 2), ("pair1", 3), ("pair1", 4), ("last_row", 0),
                                     ("last_row", 3)])
def test_small_checker_rejects_faults(fault, i):
    bh, heads, nq, nkv, hd, causal, dist = TEETH_SHAPES[i]
    q, k, v, rpb, o, bound = _teeth_case(i, *TEETH_SHAPES[i])
    assert float(ratio(emulate_small(q, k, v, heads, hd ** -0.5, causal, rpb, fault=fault), o, bound).max()) > 1.0


@pytest.mark.parametrize("T", [1, 129, 257])
def test_cls_checker_teeth(T):
    """The honest emulation passes; summing only the first 128 tokens is rejected wherever it changes anything (T > 128)."""
    g = torch.Generator().manual_seed(T)
    heads, hd = 2, 80
    q, k, v = make_qkv(g, 1, T, heads, hd, "late")
    kv = torch.cat([k, v], dim=1)
    o, sv = attn_ref(q.double(), k.double(), v.double(), heads, hd, hd ** -0.5)
    bound = attn_expect(o, sv, T, u_p=2.0 ** -22)
    assert float(ratio(emulate_cls(q, kv, heads, hd, hd ** -0.5), o, bound).max()) <= 1.0
    if T > 128:
        assert float(ratio(emulate_cls(q, kv, heads, hd, hd ** -0.5, fault="first128"), o, bound).max()) > 1.0


# ================================================================================================================ GPU: attention_small


def sa_layout(B, heads, nq, nkv, hd, causal=0, fused=False):
    """The descriptor of a GPU case (no pointers yet): every pitch with a NaN gap, batch strides with NaN gaps between images; fused:
    q, k and v are column slices of one [B, n, 3 heads hd + 8] buffer."""
    Cw = heads * hd
    if fused:
        p = 3 * Cw + 8
        d = dict(qp=p, kp=p, vp=p, qbs=nq * p + 24, kbs=nq * p + 24, vbs=nq * p + 24)
    else:
        d = dict(qp=Cw + 8, kp=Cw + 16, vp=Cw + 24, qbs=nq * (Cw + 8) + 16, kbs=nkv * (Cw + 16) + 8, vbs=nkv * (Cw + 24) + 32)
    return dict(B=B, heads=heads, nq=nq, nkv=nkv, hd=hd, causal=causal, scale=hd ** -0.5, op=Cw + 8, obs=nq * (Cw + 8) + 16, **d)


def sa_inputs(R, f, dist, fused):
    """NaN-filled flat buffers holding each image's make_qkv values at the descriptor's pitches and batch strides."""
    B, nq, nkv, heads, hd = f["B"], f["nq"], f["nkv"], f["heads"], f["hd"]
    Cw = heads * hd
    g = torch.Generator(device=R.dev).manual_seed(int(torch.randint(0, 1 << 30, (1,), generator=R.g, device=R.dev)))
    vals = [make_qkv(g, nq, nkv, heads, hd, dist, dev=R.dev) for _ in range(B)]
    if fused:
        flat = torch.full(((B - 1) * f["qbs"] + nq * f["qp"],), NAN, dtype=torch.bfloat16, device=R.dev)
        bufs = {"q": flat, "k": flat[Cw:], "v": flat[2 * Cw:]}
    else:
        bufs = {nm: torch.full(((B - 1) * f[nm + "bs"] + n_ * f[nm + "p"],), NAN, dtype=torch.bfloat16, device=R.dev)
                for nm, n_ in (("q", nq), ("k", nkv), ("v", nkv))}
    for i, nm in enumerate("qkv"):
        n_ = nq if nm == "q" else nkv
        bufs[nm].as_strided((B, n_, Cw), (f[nm + "bs"], f[nm + "p"], 1)).copy_(torch.stack([x[i] for x in vals]))
    return bufs


def _query_bufs(f, bufs, out_ptr, sms):
    return sa_query(dict(f, q=bufs["q"].data_ptr(), k=bufs["k"].data_ptr(), v=bufs["v"].data_ptr(), out=out_ptr), sms)


def run_small(R, f, dist="randn", fused=False, expect=None):
    """One GPU case: assert the plan at 132 SMs (and that it is what runs on a 132-SM device), then the census checks; -> worst."""
    bufs = sa_inputs(R, f, dist, fused)
    plan, err = _query_bufs(f, bufs, addr(9), SMS)
    assert plan is not None, err
    if expect:
        assert {k: plan[k] for k in expect} == expect, f"plan at 132 SMs {plan}, expected {expect}"
    if sms(R.dev) == SMS:
        assert _query_bufs(f, bufs, addr(9), 0)[0] == plan
    errs, (worst, where) = check_attention_small(R, f, bufs)
    assert not errs, f"{errs}; plan {plan}"
    return worst, where, plan


# (name, (B, heads, nq, nkv, hd), options, plan fields expected at 132 SMs)
SA_CASES = [
    # the row split
    ("one chunk, 33 rows per warp", (17, 16, 257, 257, 64), {}, dict(chunks=1, rows_per_block=257)),
    ("rows_per_block floor, last block 4 rows", (1, 1, 100, 100, 64), {}, dict(chunks=13, rows_per_block=8)),
    ("rows_per_block 13, last block 7 rows", (3, 4, 280, 280, 64), {}, dict(chunks=22, rows_per_block=13)),
    ("last block 1 row", (1, 2, 257, 257, 64), {}, dict(chunks=33, rows_per_block=8)),
    ("nq 1", (2, 4, 1, 50, 64), {}, dict(chunks=1, rows_per_block=8)),
    ("workload vision tower", (8, 16, 257, 257, 80), {}, dict(chunks=3, rows_per_block=86)),
    # causal: the maximum on the diagonal, 2, 3 and many chunks per head
    ("causal 77, 2 chunks", (9, 16, 77, 77, 64), dict(causal=1, dist="late"), dict(chunks=2, rows_per_block=39)),
    ("causal 77, 3 chunks (text tower)", (8, 16, 77, 77, 64), dict(causal=1, dist="late"), dict(chunks=3, rows_per_block=26)),
    ("causal 77, 10 chunks", (1, 2, 77, 77, 64), dict(causal=1, dist="late"), dict(chunks=10, rows_per_block=8)),
    ("causal 257, 2 chunks", (9, 16, 257, 257, 64), dict(causal=1, dist="late"), dict(chunks=2, rows_per_block=129)),
    ("causal 257, 3 chunks", (8, 16, 257, 257, 64), dict(causal=1, dist="late"), dict(chunks=3, rows_per_block=86)),
    ("causal 257, 33 chunks", (1, 4, 257, 257, 64), dict(causal=1, dist="late"), dict(chunks=33, rows_per_block=8)),
    ("causal 1000, 2 chunks", (2, 70, 1000, 1000, 40), dict(causal=1, dist="late"), dict(chunks=2, rows_per_block=500)),
    ("causal 1000, 3 chunks", (1, 100, 1000, 1000, 40), dict(causal=1, dist="late"), dict(chunks=3, rows_per_block=334)),
    ("causal 1000, 125 chunks", (1, 2, 1000, 1000, 40), dict(causal=1, dist="late"), dict(chunks=125, rows_per_block=8)),
    # head widths: lanes with no pair, one pair, both pairs
    *[(f"head width {hd}", (2, 3, 100, 100, hd), {}, dict(chunks=13, rows_per_block=8)) for hd in (8, 16, 40, 64, 72, 80, 120, 128)],
    # key counts
    ("nkv 1", (2, 3, 50, 1, 64), {}, dict(smem_bytes=sa_smem(64, 1))),
    *[(f"nkv {n}", (2, 3, 40, n, 64), {}, dict(smem_bytes=sa_smem(64, n))) for n in (31, 32, 33)],
    *[(f"nkv {n}, head width {hd}", (2, 3, 64, n, hd), {}, dict(smem_bytes=sa_smem(hd, n), smem_optin=1)) for n in (1023, 1024) for hd in (8, 40)],
    ("head width 128, largest nkv", (1, 2, 100, 365, 128), {}, dict(smem_bytes=204724, smem_optin=1)),
    # cross attention
    ("cross, nq 1, nkv 1024", (1, 4, 1, 1024, 40), {}, dict(chunks=1, smem_bytes=201984)),
    ("cross, nq 300, nkv 5", (2, 2, 300, 5, 64), {}, dict(chunks=38, smem_optin=0)),
    # q, k and v read in place from one fused QKV buffer
    ("fused QKV, head width 80", (3, 4, 257, 257, 80), dict(fused=True), {}),
    ("fused QKV causal, head width 64", (2, 16, 77, 77, 64), dict(fused=True, causal=1, dist="late"), {}),
    # score distributions
    ("unit scores", (2, 8, 257, 257, 80), dict(dist="unit"), {}),
    ("late maximum", (2, 8, 257, 257, 80), dict(dist="late"), {}),
    ("large logits", (2, 8, 77, 77, 64), dict(dist="large"), {}),
    ("large logits, 1024 keys", (1, 4, 64, 1024, 40), dict(dist="large"), {}),
]


@pytest.mark.gpu
@pytest.mark.parametrize("name,shape,opt,expect", SA_CASES, ids=[c[0] for c in SA_CASES])
def test_attention_small_schedule(cuda, name, shape, opt, expect):
    t0 = time.time()
    opt = dict(opt)
    f = sa_layout(*shape, causal=opt.pop("causal", 0), fused=opt.get("fused", False))
    worst, where, plan = run_small(Replay(cuda, zlib.crc32(name.encode()) & 0xFFFF), f, expect=expect, **opt)
    print(f"\n{name}: plan {plan}, worst err/bound {worst:.3g} at {where} ({time.time() - t0:.2f} s)")


@pytest.mark.gpu
def test_attention_small_optin_order(cuda):
    """A call under 48 KB, one above (the kernel's limit is raised), one under again: all three within the bound."""
    R = Replay(cuda, 48)
    for shape, optin in (((2, 4, 100, 100, 64), 0), ((2, 4, 100, 1000, 40), 1), ((2, 4, 60, 60, 80), 0)):
        f = sa_layout(*shape)
        worst, where, plan = run_small(R, f, expect=dict(smem_optin=optin))
        print(f"\n{shape}: plan {plan}, worst err/bound {worst:.3g}")


# ================================================================================================================ GPU: cls_attention
def cls_inputs(R, f, dist):
    B, T, heads, hd = f["batch"], f["tokens"], f["heads"], f["hd"]
    Cw = heads * hd
    g = torch.Generator(device=R.dev).manual_seed(int(torch.randint(0, 1 << 30, (1,), generator=R.g, device=R.dev)))
    vals = [make_qkv(g, 1, T, heads, hd, dist, dev=R.dev) for _ in range(B)]
    q0 = R.poisoned(B, f["qp"], torch.cat([x[0] for x in vals]))
    kv = R.poisoned(B * T, f["kvp"], torch.cat([torch.cat([x[1], x[2]], dim=1) for x in vals]))
    return q0, kv


# (name, (B, T, heads, hd), dist)
CLS_CASES = [
    *[(f"T {T}", (2, T, 4, 80), "randn") for T in (1, 2, 127, 128, 129, 257, 4096)],
    ("largest T at head width 80", (1, 12204, 1, 80), "randn"),
    *[(f"head width {hd}", (2, 200, 3, hd), "randn") for hd in (2, 128, 130, 256)],
    ("workload: 16 heads of 80, 9 images", (9, 257, 16, 80), "randn"),
    ("one head, one image", (1, 300, 1, 80), "randn"),
    ("late maximum", (3, 257, 4, 80), "late"),
    ("late maximum, head width 256", (2, 600, 2, 256), "late"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("name,shape,dist", CLS_CASES, ids=[c[0] for c in CLS_CASES])
def test_cls_attention_schedule(cuda, name, shape, dist):
    """q0 and out with NaN pitch gaps, kv_pitch above 2 heads hd with a NaN gap, NaN output tail rows."""
    t0 = time.time()
    B, T, heads, hd = shape
    Cw = heads * hd
    f = dict(batch=B, tokens=T, heads=heads, hd=hd, qp=Cw + 6, kvp=2 * Cw + 10, op=Cw + 4)
    R = Replay(cuda, zlib.crc32(name.encode()) & 0xFFFF)
    q0, kv = cls_inputs(R, f, dist)
    plan, err = cls_query(cls_desc(B, T, heads, hd, q=q0.data_ptr(), qp=f["qp"], kv=kv.data_ptr(), kvp=f["kvp"], out=addr(9), op=f["op"]))
    assert plan is not None and plan["smem_bytes"] == (hd + T) * 4, err
    errs, (worst, where) = check_cls(R, f, q0, kv, hd ** -0.5)
    assert not errs, errs
    print(f"\n{name}: worst err/bound {worst:.3g} at {where} ({time.time() - t0:.2f} s)")


# ================================================================================================================ GPU: placement


SA_GPU_REJECT = [("k misaligned", dict(k=8)), ("v misaligned", dict(v=4)), ("q misaligned", dict(q=2)), ("out misaligned", dict(out=2)),
                 ("q_pitch below the width", dict(qp=-16)), ("k_pitch below the width", dict(kp=-24)),
                 ("v_pitch below the width", dict(vp=-32)), ("out_pitch below the width", dict(op=-16)),
                 ("out images overlap", dict(obs=-32)), ("nkv past 200 KB at head width 128", dict(nkv=1))]


@pytest.mark.gpu
@pytest.mark.parametrize("name,delta", SA_GPU_REJECT, ids=[r[0] for r in SA_GPU_REJECT])
def test_attention_small_placement_rejected_on_device(cuda, name, delta):
    """The query rejects first; then the launching call returns the same error, launches nothing and leaves the output NaN.  Every
    pointer is an offset view into a valid allocation."""
    L = ladi_lib().load()
    R = Replay(cuda, 7)
    f = sa_layout(2, 2, 20, 365, 128)
    bufs = sa_inputs(R, f, "randn", False)
    out = torch.full((2 * f["obs"] + 64,), NAN, dtype=torch.bfloat16, device=cuda)
    a = dict(f, q=bufs["q"].data_ptr(), k=bufs["k"].data_ptr(), v=bufs["v"].data_ptr(), out=out.data_ptr())
    assert sa_query(a, 0)[0] is not None
    for k, dv in delta.items():
        a[k] += dv
    plan, err = sa_query(a, 0)
    assert plan is None and err, plan
    before = launches()
    assert L.ladi_attention_small(*[a[k] for k in SA_ORDER], None) == 1
    assert L.ladi_last_error().decode() == err
    torch.cuda.synchronize()
    assert launches() == before
    assert bool(torch.isnan(out.float()).all())


CLS_GPU_REJECT = [("kv misaligned", dict(kv=2)), ("kv_pitch below 2 heads hd", dict(kvp=-12)), ("q_pitch below heads hd", dict(qp=-8)),
                  ("out_pitch below heads hd", dict(op=-6)), ("tokens past 48 KB", dict(tokens=1))]


@pytest.mark.gpu
@pytest.mark.parametrize("name,delta", CLS_GPU_REJECT, ids=[r[0] for r in CLS_GPU_REJECT])
def test_cls_placement_rejected_on_device(cuda, name, delta):
    L = ladi_lib().load()
    R = Replay(cuda, 8)
    B, T, heads, hd = 1, 12204, 1, 80
    f = dict(batch=B, tokens=T, heads=heads, hd=hd, qp=hd + 6, kvp=2 * hd + 10, op=hd + 4)
    q0, kv = cls_inputs(R, f, "randn")
    out = R.poisoned(B + 3, f["op"])
    a = cls_desc(B, T, heads, hd, q=q0.data_ptr(), qp=f["qp"], kv=kv.data_ptr(), kvp=f["kvp"], out=out.data_ptr(), op=f["op"])
    assert cls_query(a)[0] is not None
    for k, dv in delta.items():
        a[k] += dv
    plan, err = cls_query(a)
    assert plan is None and err, plan
    before = launches()
    assert L.ladi_cls_attention(*[a[k] for k in CLS_ORDER], None) == 1
    assert L.ladi_last_error().decode() == err
    torch.cuda.synchronize()
    assert launches() == before
    assert bool(torch.isnan(out.float()).all())
