"""The float64 checking code the kernel tests share: error-bound constants, float64 references and bounds, the replay harness
(NaN-poisoned buffers, the layout check, the run-twice check), plan queries on fake addresses, the placement-rule runner, the census
machinery (trace formatter, data-flow normalisation, recording, descriptor collection), the replays more than one test file runs, and
rel_l2.  A plain module: pytest does not collect it.

The error bound is per element and is built from the error sources the kernels have.  Its constants:
  U_BF16   = 2^-7   bf16 output rounding (8-bit significand, round-to-nearest: unit roundoff 2^-8) doubled for the fp32 epilogue
                    arithmetic before it;
  U_F32    = 2^-21  fp32 output rounding (2^-24) with the same kind of margin;
  C_ACC    = 4      fp32 accumulation of K exact bf16 products (wgmma, split-K partials, fp32 norm sums): the error of a sum of K terms
                    behaves like 2^-24 * sqrt(K) * sum|terms| for rounding (and for the truncating alignment of the tensor core, whose
                    sign follows the random-walking partial sum); 4 covers the tail over millions of elements;
  SILU_REL = 2^-11  tanh.approx in SiLU (x/2 * (1 + tanh(x/2))): relative error 2^-11 of tanh, i.e. at most 2^-12 |x|, doubled;
  GELU_REL = 3e-5   the degree-8 erf polynomial of the GELU epilogue: |erf error| <= 4.8e-5 -> |gelu error| <= 2.4e-5 |x| (also past
                    the +-3 clamp, where erf(3) misses 1 by 2.2e-5);
  ACT_GAIN = 1.13   sup |act'| of SiLU (1.10) and GELU (1.13): how much an accumulation error grows through the activation;
  U_P      = 2^-7   attention: P is rounded to bf16 (2^-8) before P.V, doubled; the error it causes is at most U_P * sum p|v| / l;
  E_EXP    = 2^-16  attention: ex2.approx (2^-22 relative) plus the fp32 rounding of the exponent argument (|x| 2^-24, |x| < 2^6);
                    its domain is |x| < 2^6 for x = scale log2(e) q.k, which every attention test input keeps (EXP2_DOMAIN; attn_inputs
                    asserts it for the wgmma kernels' score distributions);
  ROUND1   = 2^-8   one round-to-nearest to bf16 (8-bit significand).
So  conv/GEMM:  |y - r| <= U * |r| + gain * C_ACC * sqrt(K) * 2^-24 * m + eps_act,  m = |A| (*) |W| + |bias| + |residual| in float64;
    attention:  |y - r| <= U * |r| + (U_P + C_ACC * sqrt(nkv) * 2^-24 + E_EXP) * sum p|v| / l   (from the float64 softmax);
    GroupNorm / LayerNorm: U * |r| + gain * |gamma| (|xhat| d_rstd + d_mean rstd) + eps_act, where the one-pass fp32 statistics give
                d_mean = delta (|mean| + std) and d_rstd = 1.5 delta (mean^2 + var) / var, delta = C_ACC sqrt(count) 2^-24: the term
                that grows with mean^2 / var, which is why the GroupNorm inputs carry per-channel offsets of a few sigma.
The bounds of the glue and front-end kernels (DDIM_ULPS, AA_POS and the references below) are derived in
tests/test_gpu_glue_frontend_census.py's docstring."""
import ctypes as C
import functools
import json
import math
import os
import re
import subprocess
import sys
from collections import OrderedDict, defaultdict

import numpy as np
import pytest
import torch
import torch.nn.functional as F

U_BF16, U_F32 = 2.0 ** -7, 2.0 ** -21
C_ACC = 4.0
SILU_REL, GELU_REL, ACT_GAIN = 2.0 ** -11, 3e-5, 1.13
U_P, E_EXP = 2.0 ** -7, 2.0 ** -16
EPS24 = 2.0 ** -24
ROUND1 = 2.0 ** -8
DDIM_ULPS = 8.0        # the DDIM update's seven fp32 roundings (CFG difference, product, sum, two products, difference, scale), plus one
AA_POS = 2.0 ** -23    # relative error of the fp32 sample position (center = scale (o + 0.5), argument (j - center + 0.5) / scale)
NAN = float("nan")
TAIL = 3  # NaN rows after an output that no call may write
SMS = 132  # the H100 SXM's SM count: the plan tables' and the CPU edge cases' device
BASE = 1 << 40  # fake device addresses for the plan queries: they dereference nothing
A = 1 << 20  # a fake, 256-byte aligned device address for the placement rules; never dereferenced


def rel_l2(y, ref):
    y, ref = y.detach().float().cpu(), ref.detach().float().cpu()
    return ((y - ref).norm() / ref.norm().clamp_min(1e-12)).item()


# ================================================================================================================ float64 references and bounds

def silu64(x):
    return x * torch.sigmoid(x)


def gelu64(x):
    return 0.5 * x * (1.0 + torch.erf(x * (0.5 ** 0.5)))


def conv_expect(pre, m, K, act, res=None, rs=None, out_fp32=False):
    """pre = A W^T + bias and m = |A| |W|^T + |bias| (+|res|), float64 [..., c_out] -> (r, bound) [..., c_eff] per the module docstring."""
    e = C_ACC * math.sqrt(K) * EPS24 * m
    if act == 2:  # GEGLU: interleaved (value, gate) columns -> value * gelu(gate)
        v, g, ev, eg = pre[..., 0::2], pre[..., 1::2], e[..., 0::2], e[..., 1::2]
        gl = gelu64(g)
        r = v * gl
        err = ev * gl.abs() + ACT_GAIN * eg * (v.abs() + ev) + GELU_REL * g.abs() * v.abs()
    else:
        if act == 1:
            r, err = silu64(pre), ACT_GAIN * e + SILU_REL * pre.abs()
        elif act == 3:
            r, err = gelu64(pre), ACT_GAIN * e + GELU_REL * pre.abs()
        elif act == 4:
            r, err = pre.clamp_min(0), e
        else:
            r, err = pre, e
        if res is not None:
            r = r + res
    if rs is not None:
        r, err = r * rs, err * rs
    return r, (U_F32 if out_fp32 else U_BF16) * r.abs() + err


def attn_expect(o, sv, nkv, u_p=None):
    """o = softmax(s) v and sv = sum p|v| / l from the float64 softmax -> bound."""
    u_p = U_P if u_p is None else u_p
    return U_BF16 * o.abs() + (u_p + C_ACC * math.sqrt(nkv) * EPS24 + E_EXP) * sv


def norm_expect(x, mean, var, gamma, beta, eps, count, silu, add=None):
    """x [..., C] float64 with mean / var broadcast to it -> (r, bound) of (x - mean) rstd gamma + beta (+SiLU) (+add)."""
    rstd = 1.0 / torch.sqrt(var + eps)
    xhat = (x - mean) * rstd
    pre = xhat * gamma + beta
    delta = C_ACC * math.sqrt(count) * EPS24
    sd = var.sqrt()
    d_mean = delta * (mean.abs() + sd)
    d_rstd = 1.5 * delta * (mean * mean + var) / (var + eps) + 2.0 ** -22
    e = gamma.abs() * (xhat.abs() * d_rstd + d_mean * rstd + 2.0 ** -23 * (x.abs() + mean.abs()) * rstd)
    if silu:
        r, e = silu64(pre), ACT_GAIN * e + SILU_REL * pre.abs()
    else:
        r = pre
    if add is not None:
        r = r + add
    return r, U_BF16 * r.abs() + e


def ratio(y, r, bound):
    """|y - r| / bound, NaN (a poisoned value that leaked into the result) -> inf."""
    q = (y.double() - r).abs() / bound.clamp_min(1e-300)
    return torch.nan_to_num(q, nan=float("inf"))


def max_ratio(y, r, bound):
    return float(ratio(y, r, bound).max())


def argworst(q):
    """-> (the largest err/bound of q, its index as a list)."""
    return float(q.max()), [int(v) for v in torch.unravel_index(q.argmax(), q.shape)]


def worst_at(q, names, extra=""):
    """err/bound q -> ([error] if it exceeds 1, (worst, where)), where = the worst element's index named by `names`."""
    w, idx = argworst(q)
    where = ", ".join(f"{n} {i}" for n, i in zip(names, idx)) + extra
    return ([f"err/bound {w:.3g} at {where}"] if w > 1 else []), (w, where)


# ================================================================================================================ the replay harness
def cpu_gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def nan_buf(shape, dtype, dev, values=None):
    """NaN over `shape`, with `values` [rows, c] in the first c columns."""
    t = torch.full(shape, NAN, dtype=dtype, device=dev)
    if values is not None:
        t[:, :values.shape[1]] = values.to(dtype)
    return t


class Replay:
    def __init__(self, dev, seed):
        self.dev = dev
        self.g = torch.Generator(device=dev).manual_seed(seed)
        self.stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def randn(self, *shape, std=1.0):
        return torch.randn(shape, device=self.dev, generator=self.g) * std

    def rand(self, *shape):
        return torch.rand(shape, device=self.dev, generator=self.g)

    def poisoned(self, rows, pitch, values=None, dtype=torch.bfloat16):
        """[rows, pitch] NaN, with `values` [rows, c] in the first c columns."""
        return nan_buf((rows, pitch), dtype, self.dev, values)


def flat_buf(R, n, dtype, tail=64, fill=NAN):
    """-> (flat buffer, first n elements): a `tail` past the end shows a write beyond the operand."""
    flat = torch.full((n + tail,), fill, dtype=dtype, device=R.dev)
    return flat, flat[:n]


def tail_nan(flat, n, what):
    t = flat[n:].float()
    return [] if bool(torch.isnan(t).all()) else [f"{what}: wrote past its end at element {n + int((~torch.isnan(t)).nonzero()[0])}"]


def layout(out, lo, hi, what, rows=None):
    """The call wrote every element of columns [lo, hi) of its first `rows` rows (finite; default all rows) and nothing else: the other
    columns and the rows after them (a tail no call may write) are still NaN."""
    o = out.view(out.shape[0], -1) if out.dim() > 2 else out
    rows = o.shape[0] if rows is None else rows
    errs = []
    own = o[:rows, lo:hi]
    if not bool(torch.isfinite(own).all()):
        errs.append(f"{what}: non-finite in its columns [{lo}, {hi}) at (row, column - {lo}) {(~torch.isfinite(own)).nonzero()[0].tolist()} "
                    "(unwritten, or a poisoned input was read)")
    for name, part in (("before", o[:rows, :lo]), ("after", o[:rows, hi:]), ("in the tail rows", o[rows:])):
        if part.numel() and not bool(torch.isnan(part.float()).all()):
            errs.append(f"{what}: wrote outside its columns [{lo}, {hi}) of rows [0, {rows}), {name} them, at (row, column) "
                        f"{(~torch.isnan(part.float())).nonzero()[0].tolist()}")
    return errs


def same(a, b):
    """Bitwise equal (floating-point values compared as their bits, so NaN payloads count)."""
    it = {torch.bfloat16: torch.int16, torch.float32: torch.int32}.get(a.dtype)
    return torch.equal(a.view(it), b.view(it)) if it is not None else torch.equal(a, b)


def twice(call, fresh):
    """fresh() -> dict of buffers; call(bufs) launches; both runs are kept for the determinism check."""
    runs = []
    for _ in range(2):
        b = fresh()
        call(b)
        runs.append(b)
    if torch.cuda.is_initialized():
        torch.cuda.synchronize()
    return runs


def determinism(runs, keys):
    return [] if all(same(runs[0][k], runs[1][k]) for k in keys) else ["two runs differ bitwise"]


def pick(n, work, limit):
    """Images the reference evaluates: all, or the first and last when the work is large."""
    return list(range(n)) if n <= 2 or work <= limit else [0, n - 1]


def ptr(t):
    return C.c_void_p(t.data_ptr() if t is not None else 0)


# ================================================================================================================ plan queries
def ladi_lib():
    from ladi_vton_b200 import lib
    return lib


def sms(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


def launches():
    return ladi_lib().load().ladi_launch_count()


def addr(slot, byte_off=0):
    return BASE + slot * (1 << 32) + byte_off


def override(a, kw):
    """a[k] = v for each k, v in kw; a key k_off adds v (a byte offset) to a[k]."""
    for k, v in kw.items():
        if k.endswith("_off"):
            a[k[:-4]] += v
        else:
            a[k] = v
    return a


def plan_query(entry, plan_type, args, fields):
    """entry(*args, &plan) -> ({field: value}, "") or (None, error message)."""
    L = ladi_lib().load()
    pl = plan_type()
    rc = getattr(L, entry)(*args, C.byref(pl))
    if rc:
        assert rc == 1, rc
        return None, L.ladi_last_error().decode()
    return {f: getattr(pl, f) for f in fields}, ""


_PLACEMENT_CHILD = r"""
import ctypes as C, json, sys
sys.path.insert(0, sys.argv[1])
from ladi_vton_b200 import lib
L = lib.load()
res = []
for name, args in json.loads(sys.argv[2]):
    fn = getattr(L, name)
    rc = fn(*[C.c_void_p(a) if t is C.c_void_p else a for a, t in zip(args, fn.argtypes)], None)
    res.append([rc, L.ladi_last_error().decode()])
print(json.dumps(res))
"""


def check_placement(table):
    """table = [(id, entry point, arguments with pointers as ints, expected message or None)], run in a child process that sees no
    device: each rule must reject with LADI_ERR_INVALID and a message naming the operand; a placement that meets the rules (None) passes
    the checks and then fails with LADI_ERR_CUDA, so no call here can launch a kernel."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    out = subprocess.run([sys.executable, "-c", _PLACEMENT_CHILD, root, json.dumps([[n, a] for _, n, a, _ in table])], env=env,
                         capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    res = json.loads(out.stdout.strip().splitlines()[-1])
    bad = []
    for (what, name, _, want), (rc, msg) in zip(table, res):
        if want is None:
            if rc != 2:
                bad.append(f"{what}: rc {rc} ({msg}); expected the checks to pass and the launch to fail without a device")
        elif rc != 1 or want not in msg:
            bad.append(f"{what}: rc {rc} ({msg}); expected LADI_ERR_INVALID with '{want}'")
    assert not bad, "\n".join(bad)


# ================================================================================================================ the census machinery
@pytest.fixture()
def record():
    from ladi_vton_b200 import lib
    lib.RECORD = []
    yield lib
    lib.RECORD = None


def recorded(fn):
    """-> the ABI calls fn() issues, recorded instead of launched (`lib.RECORD`)."""
    from ladi_vton_b200 import lib
    lib.RECORD = []
    try:
        with torch.no_grad():
            fn()
        return lib.RECORD
    finally:
        lib.RECORD = None


def cpu_pack(m, sd):
    m._sd, m.device = sd, torch.device("cpu")
    m._pack()
    m._sd = None
    return m


def check_library_defaults():
    for k in ("LADI_UP2X", "LADI_LN_FOLD", "LADI_CONV_2CTA"):  # library defaults only (the workloads run with them)
        assert k not in os.environ, f"census runs with library defaults; unset {k}"


def key_of(kind, f):
    return kind + " " + " ".join(f"{k}={v}" for k, v in f.items())


def typed(f):
    """parse()'s string fields -> numbers."""
    return {k: (float(v) if k in ("eps", "scale") else int(v)) for k, v in f.items()}


def collect(work, classify):
    """The census loop.  work = [(label, issuer, () -> items)]; classify(item) -> None (not a kernel call of the census), (kind, key,
    None, None) for a call counted under its kind but replayed by another census, or (kind, key, fields, extra dict) for a descriptor.
    -> (desc, calls): desc = OrderedDict key -> dict(kind, f, first = the issuer of its first call, n = its calls, **extra), deduplicated
    by key; calls = {label: {kind: [calls, set of keys]}}."""
    desc, calls = OrderedDict(), OrderedDict()
    for label, issuer, items in work:
        cnt = calls.setdefault(label, defaultdict(lambda: [0, set()]))
        for item in items():
            d = classify(item)
            if d is None:
                continue
            kind, key, f, extra = d
            cnt[kind][0] += 1
            if f is None:
                continue
            cnt[kind][1].add(key)
            if key not in desc:
                desc[key] = dict(kind=kind, f=f, first=issuer, n=0, **extra)
            desc[key]["n"] += 1
    return desc, calls


def assert_all_known(unknown):
    assert not unknown, "entry points recorded without a SCHEMA row (add one and a replay): " + ", ".join(sorted(set(unknown)))


def _fmt_conv(d):
    g = lambda a, i: int(a[i] or 0)
    return (f"conv k={d.ksize} s={d.stride} p={d.pad_lo} up={d.up2x} n={d.n} h={d.h_out} w={d.w_out} hin={d.h_in} win={d.w_in} cout={d.c_out} nsrc={d.n_src} "
            f"src0=@{g(d.src, 0):x} c0={d.src_c[0]} p0={d.src_pitch[0]} src1=@{g(d.src, 1):x} c1={d.src_c[1]} p1={d.src_pitch[1]} nsc={d.n_sc} "
            f"sc0=@{g(d.sc, 0):x} sc0c={d.sc_c[0]} sc0p={d.sc_pitch[0]} sc1=@{g(d.sc, 1):x} sc1c={d.sc_c[1]} sc1p={d.sc_pitch[1]} "
            f"wt=@{int(d.weight or 0):x} K={d.k_total} wp={d.weight_pitch} bias=@{int(d.bias or 0):x} bpr={d.bias_per_row} bss={d.bias_step_stride} "
            f"step=@{int(d.step_ptr or 0):x} res=@{int(d.residual or 0):x} rp={d.residual_pitch} rs=@{int(d.row_scale or 0):x} act={d.act} "
            f"out=@{int(d.out or 0):x} op={d.out_pitch} f32={d.out_fp32}")


def _v(x):
    return int(getattr(x, "value", x) or 0)


def python_trace(records):
    lines = []
    for name, a in records:
        if name == "ladi_conv2d_bf16":
            lines.append(_fmt_conv(a[0]._obj))
        elif name == "ladi_groupnorm_stats":
            lines.append(f"gn_stats x0=@{_v(a[0]):x} c0={a[1]} p0={a[2]} x1=@{_v(a[3]):x} c1={a[4]} p1={a[5]} n={a[6]} hw={a[7]} groups={a[8]}")
        elif name == "ladi_groupnorm_apply":
            lines.append(f"gn_apply x0=@{_v(a[0]):x} c0={a[1]} p0={a[2]} x1=@{_v(a[3]):x} c1={a[4]} p1={a[5]} n={a[6]} hw={a[7]} groups={a[8]} gamma=@{_v(a[10]):x} "
                         f"beta=@{_v(a[11]):x} eps={a[12]:.3g} silu={a[13]} add=@{_v(a[14]):x} ap={a[15]} out=@{_v(a[16]):x} op={a[17]}")
        elif name == "ladi_layernorm":
            lines.append(f"ln x=@{_v(a[0]):x} xp={a[1]} rows={a[2]} c={a[3]} gamma=@{_v(a[4]):x} beta=@{_v(a[5]):x} eps={a[6]:.3g} out=@{_v(a[7]):x} op={a[8]}")
        elif name in ("ladi_attention_bf16", "ladi_attention_d512_bf16"):
            d = a[0]._obj
            hd = 64 if name == "ladi_attention_bf16" else d.head_dim
            lines.append(f"attn d={hd} batch={d.batch} heads={d.heads} nq={d.nq} nkv={d.nkv} q=@{int(d.q):x} qp={d.q_pitch} qbs={d.q_batch_stride} k=@{int(d.k):x} "
                         f"kp={d.k_pitch} kbs={d.k_batch_stride} v=@{int(d.v):x} vp={d.v_pitch} vbs={d.v_batch_stride} out=@{int(d.out):x} op={d.out_pitch} "
                         f"obs={d.out_batch_stride} scale={d.scale:.6g}")
        elif name == "ladi_add_bf16":
            lines.append(f"add a=@{_v(a[0]):x} b=@{_v(a[1]):x} out=@{_v(a[2]):x} count={a[3]}")
        elif name == "ladi_upsample2x_nhwc":
            lines.append(f"upsample2x x=@{_v(a[0]):x} n={a[1]} h={a[2]} w={a[3]} c={a[4]} out=@{_v(a[5]):x}")
        elif name == "ladi_cls_attention":
            lines.append(f"cls_attn q=@{_v(a[0]):x} qp={a[1]} kv=@{_v(a[2]):x} kvp={a[3]} batch={a[4]} tokens={a[5]} heads={a[6]} hd={a[7]} out=@{_v(a[9]):x} op={a[10]}")
        elif name == "ladi_attention_small":
            v = [_v(t) for t in a]
            lines.append(f"attn_small batch={a[4]} heads={a[5]} nq={a[6]} nkv={a[7]} hd={a[8]} q=@{v[0]:x} qp={a[9]} qbs={a[13]} k=@{v[1]:x} "
                         f"kp={a[10]} kbs={a[14]} v=@{v[2]:x} vp={a[11]} vbs={a[15]} out=@{v[3]:x} op={a[12]} obs={a[16]} scale={a[17]:.6g} "
                         f"causal={a[18]}")
        else:
            lines.append(f"{name} (layout / pointwise op outside the module bodies)")
    return lines


def _out_bytes(op, f):
    """Bytes the op writes starting at its `out` address (for the data-flow normalisation)."""
    i = lambda k: int(f[k])
    if op == "conv":
        return ((i("n") * i("h") * i("w") - 1) * i("op") + (i("cout") // (2 if i("act") == 2 else 1))) * (4 if i("f32") else 2)
    if op == "gn_apply":
        return ((i("n") * i("hw") - 1) * i("op") + i("c0") + i("c1")) * 2
    if op == "ln":
        return ((i("rows") - 1) * i("op") + i("c")) * 2
    if op == "attn":
        width = i("heads") * 64 if i("d") == 64 else i("d")
        return ((i("batch") - 1) * i("obs") + (i("nq") - 1) * i("op") + width) * 2
    if op == "add":
        return i("count") * 2
    if op == "upsample2x":
        return i("n") * 4 * i("h") * i("w") * i("c") * 2
    if op == "cls_attn":
        return ((i("batch") - 1) * i("op") + i("heads") * i("hd")) * 2
    if op == "attn_small":
        return ((i("batch") - 1) * i("obs") + (i("nq") - 1) * i("op") + i("heads") * i("hd")) * 2
    return 0


def normalise(lines):
    """@address -> B<k>+off for buffers written inside the trace (youngest containing buffer), X<k> for external operands."""
    live, ext, out, nbuf = [], {}, [], 0  # live: [(start, end, id)], youngest last
    for ln in lines:
        op = ln.split(" ", 1)[0]
        f = dict(re.findall(r"(\w+)=(\S+)", ln))
        w_addr = int(f["out"][1:], 16) if "out" in f else None

        def resolve(a):
            if a == 0:
                return "NULL"
            for s, e, k in reversed(live):
                if s <= a < e:
                    return f"B{k}+{a - s}"
            if a not in ext:
                ext[a] = len(ext)
            return f"X{ext[a]}"
        toks = []
        for k, v in re.findall(r"(\w+)=(\S+)", ln):
            if v.startswith("@"):
                if k == "out":
                    continue
                toks.append(f"{k}={resolve(int(v[1:], 16))}")
            else:
                toks.append(f"{k}={v}")
        if w_addr is not None:
            size = _out_bytes(op, f)
            # every write gives birth to a buffer (no op of the module bodies writes into a slice of a buffer born inside the trace); older
            # buffers it overlaps are dead -- the C++ allocator re-uses freed workspace, torch never overlaps
            live[:] = [(s, e, k) for s, e, k in live if e <= w_addr or s >= w_addr + size]
            live.append((w_addr, w_addr + size, nbuf))
            toks.append(f"out=B{nbuf}")
            nbuf += 1
        out.append(op + " " + " ".join(toks))
    return out


def compare(py_records, cpp_trace, what):
    a = normalise(python_trace(py_records))
    b = normalise([l for l in cpp_trace.splitlines() if l.strip()])
    for i, (x, y) in enumerate(zip(a, b)):
        assert x == y, f"{what}: op {i} differs\n  python: {x}\n  c++   : {y}"
    assert len(a) == len(b), f"{what}: {len(a)} Python ops vs {len(b)} C++ ops"
    return len(a)


def parse(line):
    """-> (op, {field: value}) with every @address replaced by 1 (operand present) or 0 (absent)."""
    op = line.split(" ", 1)[0]
    f = OrderedDict()
    for k, v in re.findall(r"(\w+)=(\S+)", line):
        f[k] = ("1" if int(v[1:], 16) else "0") if v.startswith("@") else v
    return op, f


def describe(name, args, schema):
    """-> (kind, OrderedDict of fields) of one recorded call; raises KeyError for an entry point without a row in `schema`."""
    kind, spec = schema[name]
    names = spec.split()
    assert len(names) == len(args), f"{name}: {len(args)} arguments recorded, SCHEMA names {len(names)}"
    f = OrderedDict()
    for nm, a in zip(names, args):
        if nm == "stream":
            continue
        if ":" in nm:
            assert isinstance(a, C.c_void_p), f"{name}: argument {nm} is not a pointer"
            f[nm.split(":")[0]] = 1 if a.value else 0
        else:
            assert isinstance(a, (int, float)) and not isinstance(a, bool), f"{name}: argument {nm} is not a scalar"
            f[nm] = a
    return kind, f


# ================================================================================================================ the workload census
# (tests/test_gpu_workload_census.py's docstring; the glue and metrics censuses skip what it replays)
# per op: the fields the trace prints; the replay implements exactly these (an unknown op or field fails test_census_integrity)
FIELDS = {
    "conv": "k s p up n h w hin win cout nsrc src0 c0 p0 src1 c1 p1 nsc sc0 sc0c sc0p sc1 sc1c sc1p wt K wp bias bpr bss step res rp rs act out op f32",
    "gn_stats": "x0 c0 p0 x1 c1 p1 n hw groups",
    "gn_apply": "x0 c0 p0 x1 c1 p1 n hw groups gamma beta eps silu add ap out op",
    "ln": "x xp rows c gamma beta eps out op",
    "attn": "d batch heads nq nkv q qp qbs k kp kbs v vp vbs out op obs scale",
    "add": "a b out count",
    "cls_attn": "q qp kv kvp batch tokens heads hd out op",
    "timestep_embedding": "t n c kp out",
}
FIELDS = {k: v.split() for k, v in FIELDS.items()}
M_UNET, M_ENC, M_DEC, M_EMASC, M_ADAPTER, M_PLAN = 0, 1, 2, 3, 4, 5
# (workload label, [(module, batch, height, width)]): the shapes of bench.py / BASELINE.json; "ctx" = plan_context GEMM at (UNet batch) x 77 rows
WORKLOADS = [
    ("512x384, 8 images, CFG (bench default; configs 1, 2, 4)",
     [(M_UNET, 16, 64, 48), (M_ENC, 8, 512, 384), (M_DEC, 8, 64, 48), (M_EMASC, 8, 512, 384), (M_PLAN, 50, 0, 0), ("ctx", 16, 77, 1024)]),
    ("512x384, 100 DDIM steps (config 4)", [(M_PLAN, 100, 0, 0)]),
    ("1024x768, 4 images, CFG (config 3)",
     [(M_UNET, 8, 128, 96), (M_ENC, 4, 1024, 768), (M_DEC, 4, 128, 96), (M_EMASC, 4, 1024, 768), (M_PLAN, 50, 0, 0), ("ctx", 8, 77, 1024)]),
    ("one 512x384 image, CFG, 20 DDIM steps (config 0 shape)",
     [(M_UNET, 2, 64, 48), (M_ENC, 1, 512, 384), (M_DEC, 1, 64, 48), (M_EMASC, 1, 512, 384), (M_PLAN, 20, 0, 0), ("ctx", 2, 77, 1024)]),
    ("inversion adapter, 8 images x 257 tokens (inference CLI path, not in the bench)", [(M_ADAPTER, 8, 257, 0)]),
]

MODULE_NAMES = {M_UNET: "UNet", M_ENC: "VAE encode", M_DEC: "VAE decode", M_EMASC: "EMASC", M_ADAPTER: "adapter", M_PLAN: "UNet plan_steps",
                "ctx": "UNet plan_context GEMM"}


def kind_of(op, f):
    if op == "attn":
        return "attn_d64" if f["d"] == "64" else "attn_d512"
    return {"gn_apply": "gn"}.get(op, op)


def _build_engines():
    from ladi_vton_b200 import EMASC, AutoencoderKL, InversionAdapter, UNet2DConditionModel, engine as eng, synthetic as S, unet_param_shapes
    from ladi_vton_b200.vae import vae_param_shapes

    def pack(model, shapes, seed):
        model._sd = S.random_state_dict(shapes, seed, fast=True)  # the walk depends on shapes only: tiled random values are enough
        model.device = torch.device("cpu")
        model._pack()
        model._sd = None
        return model

    unet = pack(UNet2DConditionModel(), unet_param_shapes({}), 1)
    vae = pack(AutoencoderKL(), vae_param_shapes({}), 2)
    ad = pack(InversionAdapter(), InversionAdapter().param_shapes(), 4)
    ein, eout = S.emasc_channels(vae.config.block_out_channels)
    em = pack(EMASC(ein, eout), S.emasc_param_shapes(ein, eout), 3)
    W = {}
    for i, (w1, b1, w2, b2) in enumerate(em.P):
        W.update({f"emasc.{i}.w1": w1, f"emasc.{i}.b1": b1, f"emasc.{i}.w2": w2, f"emasc.{i}.b2": b2})
    engines = {M_UNET: eng.Engine(eng.flatten(unet.P), plan_only=True, **unet.engine_config()),
               M_ENC: eng.Engine(eng.flatten(vae.P), plan_only=True, **vae.engine_config()),
               M_EMASC: eng.Engine(W, plan_only=True, emasc_scales=5, emasc_in=ein, emasc_out=eout, emasc_stride=[1, 1, 2, 4, 8]),
               M_ADAPTER: eng.Engine(eng.flatten(ad.P, "adapter."), plan_only=True, adapter_dim=ad.dim, adapter_heads=ad.heads,
                                     adapter_mlp=ad.mlp_dim, adapter_hidden=ad.hidden, adapter_out=ad.out_dim)}
    engines[M_DEC], engines[M_PLAN] = engines[M_ENC], engines[M_UNET]
    return unet, engines


def _context_trace(unet, batch, tokens, dim):
    """The plan_context GEMM as the Python sequencing issues it (recorded, not launched)."""
    unet._ctx = None
    return python_trace(recorded(lambda: unet.plan_context(torch.zeros((batch, tokens, dim), dtype=torch.bfloat16))))

_CENSUS = None


def census():
    """The workload census of tests/test_gpu_workload_census.py's docstring (cached).
    -> (descriptors, calls, unparsed): descriptors = OrderedDict stripped line -> {kind, op, f, first, n}; calls = {(workload, module
    label): Counter of calls and distinct descriptors per kind}; unparsed = lines with an unknown op or field set."""
    global _CENSUS
    if _CENSUS is not None:
        return _CENSUS
    check_library_defaults()
    unet, engines = _build_engines()
    unparsed, prev = [], None

    def classify(ln):
        nonlocal prev
        op, f = parse(ln)
        if op not in FIELDS or list(f) != FIELDS[op]:
            unparsed.append(ln)
            return None
        if op == "gn_stats":  # replayed together with the gn_apply that must follow it on the same operands
            prev = f
            return None
        if op == "gn_apply":
            if prev is None or any(prev[k] != f[k] for k in FIELDS["gn_stats"]):
                unparsed.append("gn_apply without its gn_stats: " + ln)
            prev = None
        return kind_of(op, f), key_of(op, f), typed(f), dict(op=op)

    work = []
    for wl, mods in WORKLOADS:
        for mod, b, h, w in mods:
            label = f"{MODULE_NAMES[mod]} {b}x{h}x{w}" if mod not in (M_PLAN, M_ADAPTER, "ctx") else \
                {M_PLAN: f"UNet plan_steps, {b} timesteps", M_ADAPTER: f"adapter {b}x{h}", "ctx": f"plan_context GEMM, {b}x{h} rows x {w}"}[mod]
            lines = (lambda b=b, h=h, w=w: _context_trace(unet, b, h, w)) if mod == "ctx" else \
                (lambda mod=mod, b=b, h=h, w=w: [l for l in engines[mod].trace(mod, b, h, w).splitlines() if l.strip()])
            work.append(((wl, label), f"{label} [{wl}]", lines))
    desc, calls = collect(work, classify)
    _CENSUS = (desc, calls, unparsed)
    return _CENSUS


# ================================================================================================================ the glue census
TRACED = {"ladi_conv2d_bf16": "conv", "ladi_layernorm": "ln"}  # through python_trace, in the workload census's fields
MODULE_ABI = ("ladi_unet_forward", "ladi_vae_encode", "ladi_vae_decode_emasc", "ladi_emasc_forward", "ladi_inversion_adapter_forward",
              "ladi_denoise_loop")
# (label, images, height, width, guidance): bench.py's default, config 3 and config 0 shapes, and the call without guidance
PIPE_WORKLOADS = [("512x384, 8 images, CFG (bench default)", 8, 512, 384, 7.5),
                  ("1024x768, 4 images, CFG (bench config 3)", 4, 1024, 768, 7.5),
                  ("one 512x384 image, CFG (bench config 0 shape)", 1, 512, 384, 7.5),
                  ("512x384, 8 images, no guidance", 8, 512, 384, 1.0)]

FRONTEND = "inference CLI front end, 8 x 512x384 (warping, CLIP preprocess, vision tower, text tower)"


class _Stub:
    """Stands in for the pipeline's engine modules: right shapes, and only the kernels the real methods launch from Python before their
    one module-level ABI call (the workload census covers the bodies behind that call).  `AutoencoderKL.encode_nhwc` packs an NCHW input
    into a zeroed NHWC buffer of pitch 8, and `decode_nhwc` packs the latents the same way with the 1 / scaling_factor scale (vae.py);
    `UNet2DConditionModel.forward_nhwc`, `plan_context` and `EMASC.__call__` launch nothing before theirs."""

    def __init__(self, H, W):
        self.H, self.W = H, W
        self.config = type("Cfg", (), {"scaling_factor": 0.18215})()

    def encode_nhwc(self, x, nhwc=False):
        from ladi_vton_b200 import ops
        B = x.shape[0]
        if not nhwc:
            ops.nchw_to_nhwc(x.contiguous(), torch.zeros((B, self.H, self.W, 8), dtype=torch.bfloat16))
        e = lambda f, c: torch.empty((B, self.H // f, self.W // f, c), dtype=torch.bfloat16)  # noqa: E731
        return torch.empty((B, self.H // 8, self.W // 8, 8)), [None, e(1, 128), e(1, 128), e(2, 256), e(4, 512), e(8, 512)]

    def decode_nhwc(self, z, feats=None, int_layers=None, scale=1.0):
        from ladi_vton_b200 import ops
        B, _, h, w = z.shape
        ops.nchw_to_nhwc(z.contiguous(), torch.zeros((B, h, w, 8), dtype=torch.bfloat16), scale=scale)
        return torch.empty((B, self.H, self.W, 4))

    def forward_nhwc(self, x_in, step):
        return torch.empty((x_in.shape[0], x_in.shape[1], x_in.shape[2], 4))

    def plan_context(self, ctx, out=None):
        return out

    def __call__(self, sel, inv):
        return list(sel)


def _pipeline_calls(B, H, W, guidance):
    from ladi_vton_b200 import ops
    from ladi_vton_b200.pipeline import StableDiffusionTryOnePipeline as Pipe, _Session
    cfg = guidance > 1.0
    h, w = H // 8, W // 8
    stub = _Stub(H, W)
    pipe = type("PipeStub", (), {})()
    pipe.vae = pipe.unet = pipe.emasc = stub
    pipe.emasc_int_layers, pipe.vae_scale_factor, pipe.device = [1, 2, 3, 4, 5], 8, torch.device("cpu")
    s = _Session(B, 2 * B if cfg else B, h, w, H, W, 32, 18, (2 * B if cfg else B, 77, 1024), 8, torch.device("cpu"))
    s.coef = torch.zeros((50, 8))
    lay = dict(B=B, cfg=cfg, no_pose=False, cloth=True, c_mask=4, c_masked=5, c_pose=9, c_cloth=27)

    def run():
        ops.check_binarise_(s.image, s.mask, s.flags)  # _prepare_mask_and_image's device path (CUDA inputs)
        Pipe._pre(pipe, s, lay)
        Pipe._step(pipe, s, cfg, guidance)
        Pipe._post(pipe, s, lay)
    return recorded(run)


def _cpu_tower(cls, seed):
    from ladi_vton_b200 import synthetic as S
    depth = cls().config.num_hidden_layers
    t = cls(num_hidden_layers=1)
    cpu_pack(t, S.random_state_dict(t.param_shapes(), seed, fast=True))
    p0 = f"{t.prefix}.encoder.layers.0."
    for i in range(1, depth):
        t.P.update({k.replace(p0, f"{t.prefix}.encoder.layers.{i}."): v for k, v in list(t.P.items()) if k.startswith(p0)})
    t.config["num_hidden_layers"] = depth
    return t


def _frontend_calls(B=8, H=512, W=384, num_vstar=16):
    from ladi_vton_b200 import CLIPTextModel, CLIPVisionModelWithProjection, encode_text_word_embedding, generate_warped_cloth, synthetic as S
    from ladi_vton_b200.inference import StandInTokenizer, clip_pixel_values, prompts_for
    from ladi_vton_b200.warp import ConvNet_TPS, UNetVanilla
    tps, ref = ConvNet_TPS(256, 192, 21, 3), UNetVanilla(24, 3, bilinear=True)
    cpu_pack(tps, S.warp_state_dict(tps.param_shapes(), 13))
    cpu_pack(ref, S.warp_state_dict(ref.param_shapes(), 14))
    vision, text = _cpu_tower(CLIPVisionModelWithProjection, 11), _cpu_tower(CLIPTextModel, 10)
    tok = StandInTokenizer()
    ids = tok(prompts_for(["upper_body", "lower_body", "dresses", "upper_body"] * (B // 4), num_vstar), max_length=77).input_ids
    cloth = torch.zeros((B, 3, H, W))

    def run():
        generate_warped_cloth(tps, ref, cloth, torch.zeros((B, 3, H, W)), torch.zeros((B, 18, H, W)))
        vision(clip_pixel_values(cloth, torch.device("cpu")))
        encode_text_word_embedding(text, ids, torch.zeros((B, num_vstar, 1024)), num_vstar)
    return recorded(run)

_GLUE = None

# warp_grid_sample with the sampling grid DOWN-scaled, up to the factor 5 its host check allows (the CLI up-scales 256x192 -> 512x384):
# the antialiased branch of the grid resize, at an integer and at a non-integer factor
GRID_DOWNSCALE = "grid down-scaled up to the host limit (synthetic)"

SYNTHETIC = [("warp_grid_sample", OrderedDict(grid=1, gh=320, gw=240, cloth=1, n=2, c=3, H=64, W=48, out=1, op=8, c_off=0)),
             ("warp_grid_sample", OrderedDict(grid=1, gh=250, gw=235, cloth=1, n=2, c=3, H=64, W=48, out=1, op=24, c_off=21))]


def glue_collect(work):
    """work = [(workload label, () -> recorded calls)] -> (desc, calls, unknown): desc = OrderedDict key -> {kind, f, first, n} of the
    descriptors the workload census does not replay; calls = {workload: {kind: [calls, set of keys]}}; unknown = entry points recorded
    without a SCHEMA row."""
    known = census()[0]
    unknown = []

    def classify(call):
        name, args = call
        if name in MODULE_ABI:
            return None
        if name in TRACED:
            op, f = parse(python_trace([call])[0])
            return (op, key_of(op, f), None, None) if key_of(op, f) in known else (op, key_of(op, f), typed(f), {})
        if name in SCHEMA:
            kind, f = describe(name, args, SCHEMA)
            return kind, key_of(kind, f), f, {}
        unknown.append(name)
        return None
    desc, calls = collect([(wl, wl, rec) for wl, rec in work], classify)
    return desc, calls, unknown


def glue_census():
    """glue_collect() over the workloads of tests/test_gpu_glue_frontend_census.py's docstring, plus the SYNTHETIC descriptors (cached)."""
    global _GLUE
    if _GLUE is not None:
        return _GLUE
    check_library_defaults()
    work = [(wl, functools.partial(_pipeline_calls, B, H, W, g)) for wl, B, H, W, g in PIPE_WORKLOADS] + [(FRONTEND, _frontend_calls)]
    desc, calls, unknown = glue_collect(work)
    for kind, f in SYNTHETIC:
        desc[key_of(kind, f)] = dict(kind=kind, f=f, first=GRID_DOWNSCALE, n=1)
    _GLUE = (desc, calls, unknown)
    return _GLUE


# ================================================================================================================ replays
# The workload census's replay_conv / replay_ln / check_cls and the glue census's replays (bounds derived in
# tests/test_gpu_glue_frontend_census.py's docstring), which the metrics census and the schedule tests run too.
# entry point -> (kind, its arguments in order: pointers are "name:role" with role in / out / io (in place); "stream" is dropped)
SCHEMA = {
    "ladi_check_binarise": ("check_binarise", "image:in n_image mask:io n_mask flags:io stream"),
    "ladi_bilinear_down8": ("bilinear_down8", "x:in n c H W out:out stream"),
    "ladi_nchw_f32_to_nhwc_bf16": ("nchw_to_nhwc", "x:in n c h w f scale gate:in out:out op c_off stream"),
    "ladi_posterior_sample": ("posterior_sample", "mom:in mp noise:in n cz h w scale out:out stream"),
    "ladi_inv_mask_rows": ("inv_mask_rows", "mask:in n H W f out:out stream"),
    "ladi_ddim_cfg_step": ("ddim_cfg_step", "eps:in ep lat:io uin:io inp B h w cfg guidance coef:in step:io advance noise:in stream"),
    "ladi_image_out": ("image_out", "x:in f32 n h w xp out:out stream"),
    "ladi_image_out_u8": ("image_out_u8", "x:in f32 n h w xp out:out stream"),
    "ladi_resize_aa": ("resize_aa", "x:in n c h w oh ow out:out op c_off stream"),
    "ladi_clip_preprocess": ("clip_preprocess", "x:in n c h w oh ow mean:in std:in quantise out:out stream"),
    "ladi_space_to_depth2": ("space_to_depth2", "x:in n h w c xp out:out op stream"),
    "ladi_channel_affine": ("channel_affine", "x:io rows c pitch scale:in shift:in stream"),
    "ladi_l2norm_channels": ("l2norm_channels", "x:io rows c pitch stream"),
    "ladi_feature_correlation": ("feature_correlation", "fa:in fb:in n h w c out:out op stream"),
    "ladi_tps_grid": ("tps_grid", "theta:in tp inv:in rep:in n n_ctrl npts points:out grid:out stream"),
    "ladi_warp_grid_sample": ("warp_grid_sample", "grid:in gh gw cloth:in n c H W out:out op c_off stream"),
    "ladi_maxpool2_nhwc": ("maxpool2", "x:in n h w c out:out stream"),
    "ladi_upsample2x_bilinear_ac": ("upsample2x_ac", "x:in n h w c out:out stream"),
    "ladi_nhwc_f32_to_nchw_clamp": ("nhwc_to_nchw_clamp", "x:in n c h w xp lo hi out:out stream"),
    "ladi_attention_small": ("attention_small", "q:in k:in v:in out:out B heads nq nkv hd qp kp vp op qbs kbs vbs obs scale causal stream"),
    "ladi_clip_embed": ("clip_embed", "src:in tok:in wemb:in pos:in out:out rows seq c op stream"),
    "ladi_patchify": ("patchify", "px:in out:out n ch h w patch kpad stream"),
    "ladi_vit_assemble": ("vit_assemble", "patch:in pp cls:in pos:in out:out n np c stream"),
}


def conv_ref(xpad, w64, s, k, h, w):
    """float64 convolution (no padding) of xpad [nI, C, Hp, Wp] by w64 [cout, C, k, k] -> (acc, |x| (*) |w|) [nI, h, w, cout],
    im2col + GEMM in bands of output rows so no intermediate exceeds ~1 GB."""
    nI, Cin = xpad.shape[:2]
    wf = w64.reshape(w64.shape[0], -1)
    wa = wf.abs()
    xpad = xpad[:, :, :, :(w - 1) * s + k]
    acc = torch.empty((nI, h, w, wf.shape[0]), dtype=torch.float64, device=xpad.device)
    m = torch.empty_like(acc)
    band = max(1, (1 << 26) // (nI * w * wf.shape[1]))
    for y0 in range(0, h, band):
        y1 = min(h, y0 + band)
        cols = F.unfold(xpad[:, :, y0 * s:(y1 - 1) * s + k], k, stride=s)  # [nI, C k k, (y1-y0) w]
        acc[:, y0:y1] = (wf @ cols).view(nI, -1, y1 - y0, w).permute(0, 2, 3, 1)
        m[:, y0:y1] = (wa @ cols.abs_()).view(nI, -1, y1 - y0, w).permute(0, 2, 3, 1)
        del cols
    return acc, m


def attn_ref(q, k, v, heads, D, scale):
    """q [nq, heads*D], k/v [nkv, heads*D] float64 -> (o, sum p|v| / l) [nq, heads*D], chunked over queries."""
    nq, nkv = q.shape[0], k.shape[0]
    qh, kh, vh = (t.view(-1, heads, D).transpose(0, 1) for t in (q, k, v))
    o = torch.empty((heads, nq, D), dtype=torch.float64, device=q.device)
    sv = torch.empty_like(o)
    ch = max(1, (1 << 26) // (heads * nkv))
    for i in range(0, nq, ch):
        s = (qh[:, i:i + ch] @ kh.transpose(1, 2)) * scale
        p = torch.exp(s - s.amax(-1, keepdim=True))
        del s
        l = p.sum(-1, keepdim=True)
        o[:, i:i + ch] = (p @ vh) / l
        sv[:, i:i + ch] = (p @ vh.abs()) / l
        del p
    return o.transpose(0, 1).reshape(nq, heads * D), sv.transpose(0, 1).reshape(nq, heads * D)


# ================================================================================================================ flash attention: inputs, emulation
# Score distributions of the wgmma attention tests, in exp2 units x = scale log2(e) q.k (the kernels' softmax argument before the
# running maximum is subtracted).  Each stays inside the domain E_EXP is stated for, |x| < EXP2_DOMAIN (attn_inputs asserts it):
#   randn  q, k ~ N(0, 2), v ~ N(0, 1): the census's inputs; |x| reaches about 17;
#   late   the key scores rise by a step (<= 6) on every key tile, from -48 to at most +48: the maximum moves up on every tile, so l and O
#          are rescaled on every tile;
#   early  one key of tile 0 at x = 4, every other key about 40 lower: later tiles add P <= 2^-40 and alpha is exactly 1 after tile 0;
#   tail   the last key scores exactly 0 (a zero key), every other key about -6: the row maximum sits in the ragged last tile beside the
#          masked lanes, whose zero-filled keys would also score 0;
#   flat   q = 0, so every score is exactly 0: the output is the mean of V over the valid keys (v = 1 + N(0, 1/4), so the mean is far
#          from 0 and a counted padded key moves it by 1 / (nkv + 1));
#   level  scores ~ N(0, 1.5^2) around a constant offset per (image, head), the offsets spread over [-48, 48] and interleaved so that
#          consecutive (image, head) pairs, and the consecutive work items of a persistent CTA, run at very different levels.
# The structured forms (late, early, tail, level) build q = u + 0.1 n and k = t / (scale log2(e) D) u + sigma n along one sign vector u
# per head (u.u = D), so that x = t plus a few tenths of noise for a target t per key.
ATTN_DISTS = ("randn", "late", "early", "tail", "flat", "level")
EXP2_DOMAIN = 2.0 ** 6
L2E = 1.4426950408889634


def _levels(n):
    """n offsets spread over [-48, 48], in the order lowest, highest, second lowest, second highest, ..."""
    lv = torch.linspace(-48.0, 48.0, n) if n > 1 else torch.tensor([-48.0])
    order = [i // 2 if i % 2 == 0 else n - 1 - i // 2 for i in range(n)]
    return lv[order]


def score_range(q, k, heads, D, scale):
    """-> max |scale log2(e) q.k| over every head, query and key of q [nq, heads*D], k [nkv, heads*D] (float64, chunked)."""
    nq, nkv = q.shape[0], k.shape[0]
    ch = max(1, (1 << 24) // nkv)
    worst = 0.0
    for h in range(heads):
        qh, kh = q[:, h * D:(h + 1) * D].double(), k[:, h * D:(h + 1) * D].double()
        for i in range(0, nq, ch):
            worst = max(worst, float((qh[i:i + ch] @ kh.t()).abs().max()) * scale * L2E)
    return worst


def attn_inputs(dist, gen, B, heads, nq, nkv, D, scale, tile):
    """bf16 q [B, nq, heads*D], k / v [B, nkv, heads*D] with the score distribution `dist` (above) for a kernel with `tile`-key tiles,
    drawn from `gen` on its device."""
    assert dist in ATTN_DISTS, dist
    dev = gen.device
    W = heads * D
    rn = lambda *s: torch.randn(s, generator=gen, device=dev)  # noqa: E731
    if dist == "randn":
        q, k, v = (rn(B, nq, W) * 2 ** 0.5).bfloat16(), (rn(B, nkv, W) * 2 ** 0.5).bfloat16(), rn(B, nkv, W).bfloat16()
    elif dist == "flat":
        q, k, v = torch.zeros((B, nq, W), device=dev).bfloat16(), (rn(B, nkv, W) * 2 ** 0.5).bfloat16(), (1.0 + 0.5 * rn(B, nkv, W)).bfloat16()
    else:
        c = scale * L2E
        u = torch.sign(rn(1, heads, 1, D))  # [1, heads, 1, D]
        j = torch.arange(nkv, device=dev, dtype=torch.float32)
        sigma = 0.5
        if dist == "late":
            nt = -(-nkv // tile)
            t = (-48.0 + min(6.0, 96.0 / max(1, nt - 1)) * torch.div(j, tile, rounding_mode="floor")).expand(B, heads, nkv)
        elif dist == "early":
            t = torch.full((B, heads, nkv), -40.0, device=dev)
            t[..., 37 % min(nkv, tile)] = 4.0
        elif dist == "tail":
            t = torch.full((B, heads, nkv), -6.0, device=dev)
        else:  # level
            t = _levels(B * heads).to(dev).view(B, heads, 1).expand(B, heads, nkv)
            sigma = 1.0
        q = u + 0.1 * rn(B, heads, nq, D)
        k = (t[..., None] / (c * D)) * u + sigma * rn(B, heads, nkv, D)
        if dist == "early":
            k[:, :, 37 % min(nkv, tile)] = (4.0 / (c * D)) * u[:, :, 0]  # the maximum without noise: x = 4 (1 + 0.1 u.n / D)
        elif dist == "tail":
            k[:, :, nkv - 1] = 0.0
        q, k = (t_.permute(0, 2, 1, 3).reshape(B, -1, W).bfloat16() for t_ in (q, k))
        v = rn(B, nkv, W).bfloat16()
    for b in range(B):
        x = score_range(q[b], k[b], heads, D, scale)
        assert x < EXP2_DOMAIN, f"{dist}: |scale log2(e) q.k| reaches {x:.1f}, outside the domain of E_EXP"
    return q, k, v


def emulate_attn(q, k, v, scale, tile, fault=None):
    """fp32 emulation of the wgmma flash kernels for one head (q [nq, D], k / v [nkv, D] bf16) over `tile`-key tiles (128 for
    attention_d64_kernel, 64 for attention_kernel<D>), in the kernels' arrangement: a query row lives in the 4 lanes of a quad, lane j
    holding keys and output columns with (index mod 8) // 2 == j; each lane keeps the running maximum m (exp2 units), its partial row
    sum l from the fp32 P, and its O columns, which P rounded to bf16 times V accumulates into.  Per tile: m' = max(m, tile row max),
    alpha = exp2(m - m'), P = exp2(s scale log2(e) - m'), l = alpha l + sum P, O = alpha O + P V.  The output is O / (sum of the 4 l).
    The faults:
      "padded"  every padded key of the last tile (zero-filled K and V: score 0) enters the softmax;
      "mask"    the ragged mask is off by one and admits key nkv (zero-filled: score 0);
      "l" / "o" a new running maximum does not rescale l / O;
      "late"    the alpha of tile j + 1 is applied before P_j V_j is added, so P_j V_j escapes one rescale;
      "quad"    the running maximum is taken per lane, without the reduction over the quad."""
    nq, D = q.shape
    nkv = k.shape[0]
    nt = -(-nkv // tile)
    kp = torch.zeros((nt * tile, D), dtype=torch.float32)
    vp = torch.zeros_like(kp)
    kp[:nkv], vp[:nkv] = k.float(), v.float()
    valid = nt * tile if fault == "padded" else nkv + 1 if fault == "mask" else nkv
    lane_k, lane_c = (torch.arange(tile) % 8) // 2, (torch.arange(D) % 8) // 2
    c = float(torch.tensor(scale, dtype=torch.float32) * torch.tensor(L2E, dtype=torch.float32))  # scale_log2, rounded to fp32
    m = torch.full((nq, 4), -float("inf"))
    l = torch.zeros((nq, 4))
    acc = torch.zeros((nq, D))
    pend = torch.zeros((nq, D))
    for t in range(nt):
        s = q.float() @ kp[t * tile:(t + 1) * tile].t()
        s[:, torch.arange(t * tile, (t + 1) * tile) >= valid] = -float("inf")
        mx = torch.stack([s[:, lane_k == j].amax(1) for j in range(4)], 1) * c
        if fault != "quad":
            mx = mx.amax(1, keepdim=True).expand(-1, 4)
        mn = torch.maximum(m, mx)
        alpha = torch.exp2(m - mn)
        p = torch.exp2(s * c - mn[:, lane_k])
        psum = torch.stack([p[:, lane_k == j].sum(1) for j in range(4)], 1)
        l = (l if fault == "l" else l * alpha) + psum
        pv = p.bfloat16().float() @ vp[t * tile:(t + 1) * tile]
        if fault == "o":
            acc = acc + pv
        elif fault == "late":
            acc, pend = acc * alpha[:, lane_c] + pend, pv
        else:
            acc = acc * alpha[:, lane_c] + pv
        m = mn
    return ((acc + pend) / l.sum(1, keepdim=True)).bfloat16()


def _lpd(v, cap):
    d = 1
    while d * 2 <= cap and v % (d * 2) == 0:
        d *= 2
    return d


def _m_tile(f, img, y, x):
    up, k, s = f["up"], f["k"], f["s"]
    HO, WO = (f["h"] // 2, f["w"] // 2) if up else (f["h"], f["w"])
    yy, xx = (y // 2, x // 2) if up else (y, x)
    bw = 128 if (k == 1 and f["h"] == 1 and s == 1) else _lpd(WO, 128)
    bh = _lpd(HO, 128 // bw)
    bn = 128 // (bw * bh)
    tx, ty = -(-WO // bw), -(-HO // bh)
    t = ((img // bn) * ty + yy // bh) * tx + xx // bw
    par = f" parity ({y % 2}, {x % 2})" if up else ""
    return f"M tile {t} of {tx * ty * -(-f['n'] // bn)}{par} (tile = {bn} x {bh} x {bw} pixels)"


def replay_conv(R, f):
    from ladi_vton_b200 import lib, ops, weights
    n, h, w, cout, k, s, pad, up, act = (f[x] for x in ("n", "h", "w", "cout", "k", "s", "p", "up", "act"))
    hin, win, K = f["hin"], f["win"], f["K"]
    srcs = [(f["c0"], f["p0"]), (f["c1"], f["p1"])][:f["nsrc"]]
    scs = [(f["sc0c"], f["sc0p"]), (f["sc1c"], f["sc1p"])][:f["nsc"]]
    rows = n * h * w
    c_eff = cout // 2 if act == 2 else cout
    xs = [R.poisoned(n * hin * win, p, R.randn(n * hin * win, c)) for c, p in srcs]
    sc = [R.poisoned(rows, p, R.randn(rows, c)) for c, p in scs]
    csum, scsum = sum(c for c, _ in srcs), sum(c for c, _ in scs)
    fan = k * k * csum + scsum
    wmain = R.randn(cout, csum, k, k, std=fan ** -0.5).bfloat16().float()
    wsc = R.randn(cout, scsum, std=fan ** -0.5).bfloat16().float() if scs else None
    if up:
        packed = weights.pack_conv_up2x(wmain, [c for c, _ in srcs])
        wref = weights.merge_up2x(wmain).bfloat16().double()  # what the kernel multiplies: the merged 2x2 weights, rounded once
    else:
        packed = weights.pack_conv(wmain, [c for c, _ in srcs], wsc[:, :, None, None] if scs else None, [c for c, _ in scs])
    assert packed.shape[1] == K, f"packed K {packed.shape[1]} != descriptor K {K}"
    wbuf = R.poisoned(packed.shape[0], f["wp"], packed)
    step = bias_eff = bias_buf = None
    if f["bias"]:
        if f["bpr"]:
            bias_buf = R.randn(rows)
            bias_eff = bias_buf[:, None]
        elif f["bss"]:  # per-step bias table: the kernel adds *step_ptr * stride; the engine points into the middle of the table
            tab = R.randn(4, f["bss"], std=0.5)
            off = (f["bss"] - cout) // 2 // 4 * 4
            step = torch.tensor([2, 0], dtype=torch.int32, device=R.dev)
            bias_buf, bias_eff = tab.view(-1)[off:], tab[2, off:off + cout]
        else:
            bias_buf = bias_eff = R.randn(cout, std=0.5)
    res = R.poisoned(rows, f["rp"], R.randn(rows, cout)) if f["res"] else None
    rs = R.rand(rows) if f["rs"] else None
    odt = torch.float32 if f["f32"] else torch.bfloat16
    ws = torch.empty(ops.SPLITK_WS_BYTES // 4, dtype=torch.float32, device=R.dev)

    d = lib.ConvDesc()
    for fld, key in (("n", "n"), ("h_out", "h"), ("w_out", "w"), ("c_out", "cout"), ("h_in", "hin"), ("w_in", "win"), ("ksize", "k"), ("stride", "s"),
                     ("pad_lo", "p"), ("n_src", "nsrc"), ("n_sc", "nsc"), ("k_total", "K"), ("weight_pitch", "wp"), ("bias_per_row", "bpr"),
                     ("bias_step_stride", "bss"), ("residual_pitch", "rp"), ("act", "act"), ("out_pitch", "op"), ("out_fp32", "f32"), ("up2x", "up")):
        setattr(d, fld, f[key])
    for i, (c, p) in enumerate(srcs):
        d.src[i], d.src_c[i], d.src_pitch[i] = xs[i].data_ptr(), c, p
    for i, (c, p) in enumerate(scs):
        d.sc[i], d.sc_c[i], d.sc_pitch[i] = sc[i].data_ptr(), c, p
    d.weight = wbuf.data_ptr()
    d.bias = bias_buf.data_ptr() if bias_buf is not None else None
    d.step_ptr = step.data_ptr() if step is not None else None
    d.residual = res.data_ptr() if res is not None else None
    d.row_scale = rs.data_ptr() if rs is not None else None
    d.splitk_ws, d.splitk_ws_bytes = ws.data_ptr(), ops.SPLITK_WS_BYTES

    def call(b):
        d.out = b["out"].data_ptr()
        lib.call("ladi_conv2d_bf16", C.byref(d), R.stream)
    runs = twice(call, lambda: dict(out=R.poisoned(rows, f["op"], dtype=odt)))
    outs = [r["out"] for r in runs]
    errs = layout(outs[0], 0, c_eff, "output") + determinism(runs, ["out"])
    if errs:
        return errs, None

    imgs = pick(n, n * h * w * cout * K, 1 << 35)
    sel = torch.tensor(imgs, device=R.dev)
    nI = len(imgs)
    X = torch.cat([x.view(n, hin, win, -1)[sel, ..., :c].double() for x, (c, _) in zip(xs, srcs)], dim=3).permute(0, 3, 1, 2)
    if up:
        xpad = F.pad(X, (1, 1, 1, 1))
        acc = torch.empty((nI, h, w, cout), dtype=torch.float64, device=R.dev)
        m = torch.empty_like(acc)
        for p in range(4):
            py, px = p // 2, p % 2
            a_, m_ = conv_ref(xpad[:, :, py:py + hin + 1, px:px + win + 1], wref[p], 1, 2, hin, win)
            acc[:, py::2, px::2], m[:, py::2, px::2] = a_, m_
    else:
        pe = pad if k == 3 else 0
        xpad = F.pad(X, (pe, max(0, (w - 1) * s + k - pe - win), pe, max(0, (h - 1) * s + k - pe - hin)))
        acc, m = conv_ref(xpad, wmain.double(), s, k, h, w)
    del X, xpad
    if scs:
        Sx = torch.cat([t.view(n, h, w, -1)[sel, ..., :c].double() for t, (c, _) in zip(sc, scs)], dim=3)
        acc += Sx @ wsc.double().t()
        m += Sx.abs() @ wsc.double().abs().t()
        del Sx
    if bias_eff is not None:
        be = bias_eff.double()
        if f["bpr"]:
            be = be.view(n, h, w, 1)[sel]
        acc += be
        m += be.abs()
    rsel = res.view(n, h, w, -1)[sel, ..., :cout].double() if res is not None else None
    if rsel is not None:
        m += rsel.abs()
    rss = rs.view(n, h, w, 1)[sel].double() if rs is not None else None
    r, bound = conv_expect(acc, m, K, act, rsel, rss, bool(f["f32"]))
    del acc, m
    y = outs[0].view(n, h, w, -1)[sel, ..., :c_eff]
    q = ratio(y, r, bound)
    worst = float(q.max())
    i0, yy, xx, cc = (int(v) for v in torch.unravel_index(q.argmax(), q.shape))
    ac = 2 * cc if act == 2 else cc
    where = (f"image {imgs[i0]}, y {yy}, x {xx}, channel {cc}: {_m_tile(f, imgs[i0], yy, xx)}, accumulator columns [{ac // 64 * 64}, "
             f"{ac // 64 * 64 + 64}) (N tile {ac // 128} at BN 128, {ac // 64} at BN 64); got {float(y[i0, yy, xx, cc]):.6g}, "
             f"ref {float(r[i0, yy, xx, cc]):.6g}, bound {float(bound[i0, yy, xx, cc]):.3g}")
    return ([f"err/bound {worst:.3g} at {where}"] if worst > 1 else []), (worst, where)


def check_cls(R, f, q0, kv, scale):
    """Run the descriptor f twice on q0 [B, qp] and kv [B * T, kvp] (NaN in their pitch gaps) into a NaN-poisoned output with TAIL
    extra rows, then check the layout, determinism and the float64 bound."""
    from ladi_vton_b200 import lib
    B, T, heads, hd = f["batch"], f["tokens"], f["heads"], f["hd"]
    Cw = heads * hd
    runs = twice(lambda b: lib.call("ladi_cls_attention", ptr(q0), f["qp"], ptr(kv), f["kvp"], B, T, heads, hd, scale, ptr(b["out"]), f["op"],
                                    R.stream), lambda: dict(out=R.poisoned(B + TAIL, f["op"])))
    outs = [r["out"] for r in runs]
    errs = layout(outs[0], 0, Cw, "output", rows=B) + determinism(runs, ["out"])
    if errs:
        return errs, None
    worst, where = 0.0, ""
    for b in range(B):
        kvb = kv[b * T:(b + 1) * T].double()
        o, sv = attn_ref(q0[b:b + 1, :Cw].double(), kvb[:, :Cw], kvb[:, Cw:2 * Cw], heads, hd, scale)
        qq = ratio(outs[0][b:b + 1, :Cw], o, attn_expect(o, sv, T, u_p=2.0 ** -22))  # P stays fp32 in this kernel
        if float(qq.max()) > worst:
            c = int(qq.argmax())
            worst, where = float(qq.max()), f"image {b}, head {c // hd}, column {c % hd}"
    return ([f"err/bound {worst:.3g} at {where}"] if worst > 1 else []), (worst, where)


def norm_input(R, rows, c):
    """bf16 values with per-channel scales and offsets of a few sigma (the regime where one-pass fp32 variance loses digits)."""
    return (R.randn(rows, c) * torch.exp(R.randn(c, std=0.5)) + R.randn(c, std=3.0)).bfloat16()


def replay_ln(R, f):
    from ladi_vton_b200 import lib
    rows, c = f["rows"], f["c"]
    x = R.poisoned(rows, f["xp"], norm_input(R, rows, c))
    gamma, beta = 1.0 + R.randn(c, std=0.25), R.randn(c, std=0.25)
    runs = twice(lambda b: lib.call("ladi_layernorm", ptr(x), f["xp"], rows, c, ptr(gamma), ptr(beta), f["eps"], ptr(b["out"]), f["op"], R.stream),
                 lambda: dict(out=R.poisoned(rows, f["op"])))
    errs = layout(runs[0]["out"], 0, c, "output") + determinism(runs, ["out"])
    if errs:
        return errs, None
    xd = x[:, :c].double()
    mean = xd.mean(dim=1, keepdim=True).expand_as(xd)
    var = xd.var(dim=1, unbiased=False, keepdim=True).expand_as(xd)
    r, bound = norm_expect(xd, mean, var, gamma.double(), beta.double(), f["eps"], c, False)
    return worst_at(ratio(runs[0]["out"][:, :c], r, bound), ("row", "column"))


@functools.lru_cache(maxsize=None)
def aa_weights(n_in, n_out):
    """torch's antialiased bilinear filter (aten upsample_bilinear2d_aa, align_corners=False), restated in float64 -> (W [n_out, n_in],
    E [n_out, n_in]): W the normalised triangle weights, E a bound on the absolute error of the kernel's fp32 weights over the window
    widened by one tap on each side (a position error can move a tap across the window's truncated edge, where its weight is ~0)."""
    scale = n_in / n_out
    support = max(scale, 1.0)
    inv = 1.0 / scale if scale >= 1.0 else 1.0
    Wm, E = torch.zeros((n_out, n_in), dtype=torch.float64), torch.zeros((n_out, n_in), dtype=torch.float64)
    for o in range(n_out):
        center = scale * (o + 0.5)
        lo, hi = max(int(center - support + 0.5), 0), min(int(center + support + 0.5), n_in)  # int() truncates toward zero, as aten
        j = torch.arange(lo, hi, dtype=torch.float64)
        wt = (1.0 - ((j - center + 0.5) * inv).abs()).clamp_min(0.0)
        tot = float(wt.sum())
        Wm[o, lo:hi] = wt / tot
        d = AA_POS * (center + support + 2.0) * inv + 2.0 ** -22
        E[o, max(lo - 1, 0):min(hi + 1, n_in)] = (hi - lo + 2) * d / tot
    return Wm, E


def resample_expect(x, oh, ow, u_out):
    """x [..., h, w] float64 -> (r, bound) of the separable antialiased resize to (oh, ow), per the module docstring."""
    Wy, Ey = (t.to(x.device) for t in aa_weights(x.shape[-2], oh))
    Wx, Ex = (t.to(x.device) for t in aa_weights(x.shape[-1], ow))
    taps = int((Wy != 0).sum(1).max()) + int((Wx != 0).sum(1).max()) + 2
    r = Wy @ x @ Wx.t()
    ax = x.abs()
    err = (taps * EPS24) * (Wy @ ax @ Wx.t()) + Ey @ ax @ Wx.t() + Wy @ ax @ Ex.t() + Ey @ ax @ Ex.t()
    return r, u_out * r.abs() + err


def corr_expect(fa, fb):
    """fa, fb NHWC [n, h, w, c] float64 -> (r, bound) NHWC [n, h, w, h*w]: FeatureCorrelation of ConvNet_TPS.py as written there
    (feature_A transposed to (w, h) order, bmm, view, two transposes), seen channels-last."""
    def corr(a, b):
        n, h, w, c = a.shape
        A, B = a.permute(0, 3, 1, 2), b.permute(0, 3, 1, 2)
        feature_A = A.transpose(2, 3).contiguous().view(n, c, h * w)
        feature_B = B.contiguous().view(n, c, h * w).transpose(1, 2)
        mul = torch.bmm(feature_B, feature_A)
        return mul.view(n, h, w, h * w).transpose(2, 3).transpose(1, 2).permute(0, 2, 3, 1)
    r, m = corr(fa, fb), corr(fa.abs(), fb.abs())
    return r, U_BF16 * r.abs() + C_ACC * math.sqrt(fa.shape[3]) * EPS24 * m


def small_attn_expect(q, k, v, heads, scale, causal):
    """q [nq, C], k / v [nkv, C] float64 -> (o, bound) [nq, C]; the causal mask (key j visible to query i iff j <= i) is applied here."""
    nq, nkv, Cw = q.shape[0], k.shape[0], q.shape[1]
    hd = Cw // heads
    qh, kh, vh = (t.view(-1, heads, hd).transpose(0, 1) for t in (q, k, v))
    s = (qh @ kh.transpose(1, 2)) * scale
    if causal:
        s = s.masked_fill(torch.ones((nq, nkv), dtype=torch.bool, device=q.device).triu(1), -float("inf"))
    p = torch.exp(s - s.amax(-1, keepdim=True))
    l = p.sum(-1, keepdim=True)
    o = ((p @ vh) / l).transpose(0, 1).reshape(nq, Cw)
    sv = ((p @ vh.abs()) / l).transpose(0, 1).reshape(nq, Cw)
    return o, attn_expect(o, sv, nkv, u_p=2.0 ** -22)


def ddim_expect(x, eu, et, row, g, cfg, noise=None):
    """One DDIM step (+CFG) in float64 on [B, 4, h, w] tensors; row = the fp32 coefficient row {1/sqrt(a), sqrt(1-a), sqrt(a_prev),
    sqrt(1-a_prev-sigma^2), sigma} -> (r, bound)."""
    inv_sa, s1a, sap, s1ap, sigma = (float(v) for v in row[:5])
    e = eu + g * (et - eu) if cfg else eu
    r = sap * (x - s1a * e) * inv_sa + s1ap * e
    E = eu.abs() + (g * (et - eu).abs() + e.abs() if cfg else 0.0)
    M = abs(sap * inv_sa) * (x.abs() + abs(s1a) * E) + abs(s1ap) * E
    if noise is not None:
        r = r + sigma * noise
        M = M + abs(sigma) * noise.abs()
    return r, DDIM_ULPS * EPS24 * M + EPS24 * r.abs()


def warp_expect(low_grid, cloth, u_out=U_BF16):
    """low_grid [n, gh, gw, 2], cloth [n, c, H, W] float64 -> (r, bound) [n, c, H, W]: antialiased resize of the grid to (H, W), then
    grid_sample(bilinear, padding_mode='border', align_corners=False)."""
    n, c, H, W = cloth.shape
    g, eg = resample_expect(low_grid.permute(0, 3, 1, 2), H, W, 2.0 ** -24)  # [n, 2, H, W]; fp32 grid, no further rounding
    gx, gy = g[:, 0], g[:, 1]
    ix = (((gx + 1.0) * W - 1.0) * 0.5).clamp(0.0, W - 1.0)
    iy = (((gy + 1.0) * H - 1.0) * 0.5).clamp(0.0, H - 1.0)
    dix = eg[:, 0] * W * 0.5 + 3 * EPS24 * ((gx.abs() + 1.0) * W * 0.5 + 1.0)
    diy = eg[:, 1] * H * 0.5 + 3 * EPS24 * ((gy.abs() + 1.0) * H * 0.5 + 1.0)
    x0, y0 = ix.floor(), iy.floor()
    wx1, wy1 = ix - x0, iy - y0
    x0, y0 = x0.long(), y0.long()
    x1, y1 = (x0 + 1).clamp_max(W - 1), (y0 + 1).clamp_max(H - 1)
    flat = cloth.reshape(n, c, H * W)
    at = lambda yy, xx: torch.gather(flat, 2, (yy * W + xx).view(n, 1, -1).expand(n, c, -1)).view(n, c, H, W)  # noqa: E731
    w00, w01, w10, w11 = ((1 - wy1) * (1 - wx1))[:, None], ((1 - wy1) * wx1)[:, None], (wy1 * (1 - wx1))[:, None], (wy1 * wx1)[:, None]
    v00, v01, v10, v11 = at(y0, x0), at(y0, x1), at(y1, x0), at(y1, x1)
    r = w00 * v00 + w01 * v01 + w10 * v10 + w11 * v11
    m = w00 * v00.abs() + w01 * v01.abs() + w10 * v10.abs() + w11 * v11.abs()
    # how far the value moves per texel of position error: the largest neighbouring difference within one texel of the sample
    dX = F.max_pool2d(F.pad((cloth[..., 1:] - cloth[..., :-1]).abs(), (0, 1)), 3, 1, 1).reshape(n, c, H * W)
    dY = F.max_pool2d(F.pad((cloth[..., 1:, :] - cloth[..., :-1, :]).abs(), (0, 0, 0, 1)), 3, 1, 1).reshape(n, c, H * W)
    lx = torch.maximum(*(torch.gather(dX, 2, (yy * W + x0).view(n, 1, -1).expand(n, c, -1)) for yy in (y0, y1))).view(n, c, H, W)
    ly = torch.maximum(*(torch.gather(dY, 2, (y0 * W + xx).view(n, 1, -1).expand(n, c, -1)) for xx in (x0, x1))).view(n, c, H, W)
    return r, u_out * r.abs() + 4 * EPS24 * m + dix[:, None] * lx + diy[:, None] * ly


def upsample_ac_expect(x):
    """x NHWC [n, h, w, c] float64 -> (r, bound) NHWC [n, 2h, 2w, c] of bilinear 2x upsampling with align_corners=True."""
    n, h, w, c = x.shape

    def axis(size):
        pos = torch.arange(2 * size, dtype=torch.float64, device=x.device) * ((size - 1) / (2 * size - 1))
        i0 = pos.floor().long()
        return i0, (i0 + 1).clamp_max(size - 1), pos - i0, 2.0 ** -22 * pos + 2.0 ** -23
    y0, y1, wy, dy = axis(h)
    x0, x1, wx, dx = axis(w)
    g = lambda yy, xx: x[:, yy][:, :, xx]  # noqa: E731
    wy_, wx_ = wy.view(1, -1, 1, 1), wx.view(1, 1, -1, 1)
    v00, v01, v10, v11 = g(y0, x0), g(y0, x1), g(y1, x0), g(y1, x1)
    r = (1 - wy_) * ((1 - wx_) * v00 + wx_ * v01) + wy_ * ((1 - wx_) * v10 + wx_ * v11)
    m = (1 - wy_) * ((1 - wx_) * v00.abs() + wx_ * v01.abs()) + wy_ * ((1 - wx_) * v10.abs() + wx_ * v11.abs())
    lx = torch.maximum((v01 - v00).abs(), (v11 - v10).abs())
    ly = torch.maximum((v10 - v00).abs(), (v11 - v01).abs())
    # the position error stays below one texel, and within [i0, i0 + 1] the interpolant's slope is the neighbour difference
    return r, U_BF16 * r.abs() + 6 * EPS24 * m + dy.view(1, -1, 1, 1) * ly + dx.view(1, 1, -1, 1) * lx


def exact(y, r, what):
    """bit-exact comparison (NaN allowed where the reference has it, whatever its payload) -> ([error], (0 or inf, where))."""
    if same(y.contiguous(), r.contiguous()):
        return [], (0.0, "bit-exact")
    it = {torch.bfloat16: torch.int16, torch.float32: torch.int32}.get(y.dtype)
    bad = (y.contiguous().view(it) != r.contiguous().view(it)) if it is not None else (y != r)
    if it is not None:
        bad &= ~(torch.isnan(y) & torch.isnan(r))
        if not bool(bad.any()):
            return [], (0.0, "bit-exact, NaN where the reference has NaN")
    loc = [int(v) for v in bad.nonzero()[0]]
    msg = f"{what}: {int(bad.sum())} elements differ; first at index {loc}: got {y[tuple(loc)].item()}, ref {r[tuple(loc)].item()}"
    return [msg], (float("inf"), msg)


def _image(R, *shape):
    return R.rand(*shape) * 2 - 1


def _binary_mask(R, *shape):
    """{0, 1} with a sprinkle of exactly 0.5 (the value the `< 0.5` comparisons must send to the masked side)."""
    m = (R.rand(*shape) < 0.4).float()
    return torch.where(R.rand(*shape) < 0.02, torch.full_like(m, 0.5), m)


def replay_nchw_to_nhwc(R, f, gate_nan=False):
    from ladi_vton_b200 import lib
    n, c, h, w, fct, op, c_off = f["n"], f["c"], f["h"], f["w"], f["f"], f["op"], f["c_off"]
    H, W = h * fct, w * fct
    x = _image(R, n, c, H, W) if f["scale"] == 1.0 else R.randn(n, c, H, W)  # scale != 1: the latents the VAE decoder loads
    gate = _binary_mask(R, n, 1, H, W) if f["gate"] else None
    if gate is not None and gate_nan:  # NaN < 0.5 is false: a NaN gate masks the pixel, as `image * (mask < 0.5)` does
        gate = torch.where(R.rand(n, 1, H, W) < 0.05, NAN, gate)
    rows = n * h * w

    def fresh():
        flat, o = flat_buf(R, rows * op, torch.bfloat16)
        return dict(flat=flat, out=o)
    runs = twice(lambda b: lib.call("ladi_nchw_f32_to_nhwc_bf16", ptr(x), n, c, h, w, fct, f["scale"], ptr(gate), ptr(b["out"]), op, c_off, R.stream),
                 fresh)
    out = runs[0]["out"].view(rows, op)
    errs = layout(out, c_off, c_off + c, "output") + tail_nan(runs[0]["flat"], rows * op, "output") + determinism(runs, ["flat"])
    # the kernel rounds the fp32 product x * scale to bf16: bit-equal to that, and (exact product when scale = 1; for the decoder's
    # 1 / scaling_factor the fp32 product carries 2^-24 before the bf16 rounding) within ROUND1 (1 + 2^-15) of float64
    xs = x[:, :, ::fct, ::fct]
    v, r = xs * f["scale"], xs.double() * float(np.float32(f["scale"]))
    if gate is not None:  # a masked pixel is +0 (`image * (mask < 0.5)` gives -0 for a negative pixel: the same value)
        keep = gate[:, :, ::fct, ::fct] < 0.5
        v, r = torch.where(keep, v, 0.0), torch.where(keep, r, 0.0)
    y = out[:, c_off:c_off + c].contiguous()
    e, res = exact(y, v.permute(0, 2, 3, 1).reshape(rows, c).bfloat16(), "values against bf16(fp32 product)")
    r = r.permute(0, 2, 3, 1).reshape(rows, c)
    e2, res2 = worst_at(ratio(y, r, ROUND1 * (1 + 2.0 ** -15) * r.abs()), ("pixel", "channel"))
    return errs + e + e2, (res if e else res2)


def replay_nhwc_to_nchw_clamp(R, f, values=None):
    from ladi_vton_b200 import lib
    n, c, h, w, xp, lo, hi = f["n"], f["c"], f["h"], f["w"], f["xp"], f["lo"], f["hi"]
    x = R.poisoned(n * h * w, xp, R.randn(n * h * w, c) * 0.8 if values is None else values, dtype=torch.float32)

    def fresh():
        flat, o = flat_buf(R, n * c * h * w, torch.float32)
        return dict(flat=flat, out=o)
    runs = twice(lambda b: lib.call("ladi_nhwc_f32_to_nchw_clamp", C.c_void_p(x.data_ptr()), n, c, h, w, xp, lo, hi, C.c_void_p(b["out"].data_ptr()),
                                     R.stream), fresh)
    errs = tail_nan(runs[0]["flat"], n * c * h * w, "output") + determinism(runs, ["flat"])
    ref = x[:, :c].reshape(n, h, w, c).permute(0, 3, 1, 2).clamp(lo, hi).contiguous().view(-1)  # torch.clamp keeps NaN
    e, res = exact(runs[0]["out"], ref, "values")
    return errs + e, res


def replay_inv_mask_rows(R, f):
    from ladi_vton_b200 import lib
    n, H, W, fct = f["n"], f["H"], f["W"], f["f"]
    mask = _binary_mask(R, n, 1, H, W)
    cnt = n * (H // fct) * (W // fct)

    def fresh():
        flat, o = flat_buf(R, cnt, torch.float32)
        return dict(flat=flat, out=o)
    runs = twice(lambda b: lib.call("ladi_inv_mask_rows", C.c_void_p(mask.data_ptr()), n, H, W, fct, C.c_void_p(b["out"].data_ptr()), R.stream), fresh)
    errs = tail_nan(runs[0]["flat"], cnt, "output") + determinism(runs, ["flat"])
    e, res = exact(runs[0]["out"], (1.0 - mask[:, 0, ::fct, ::fct]).reshape(-1), "values")
    return errs + e, res


def replay_bilinear_down8(R, f):
    from ladi_vton_b200 import lib
    n, c, H, W = f["n"], f["c"], f["H"], f["W"]
    x = R.rand(n, c, H, W) ** 4  # pose-map-like: mostly small, peaks near 1
    cnt = n * c * (H // 8) * (W // 8)

    def fresh():
        flat, o = flat_buf(R, cnt, torch.float32)
        return dict(flat=flat, out=o)
    runs = twice(lambda b: lib.call("ladi_bilinear_down8", C.c_void_p(x.data_ptr()), n, c, H, W, C.c_void_p(b["out"].data_ptr()), R.stream), fresh)
    errs = tail_nan(runs[0]["flat"], cnt, "output") + determinism(runs, ["flat"])
    y = runs[0]["out"].view(n, c, H // 8, W // 8)
    e, _ = exact(y, F.interpolate(x, size=(H // 8, W // 8), mode="bilinear", align_corners=False), "against fp32 F.interpolate")
    q = x.double()[:, :, 3::8, 3::8], x.double()[:, :, 3::8, 4::8], x.double()[:, :, 4::8, 3::8], x.double()[:, :, 4::8, 4::8]
    r = 0.25 * sum(q)
    errs2, res = worst_at(ratio(y, r, 2.0 ** -23 * 0.25 * sum(t.abs() for t in q)), ("image", "channel", "y", "x"))
    return errs + e + errs2, res


def replay_check_binarise(R, f):
    from ladi_vton_b200 import lib
    ni, nm = f["n_image"], f["n_mask"]
    image_flat, image = flat_buf(R, ni, torch.float32, fill=5.0)  # a read past the end would raise the image flag
    image.copy_(_image(R, ni))
    image[::7919] = NAN  # NaN compares false: no flag, as the reference's min / max test
    m0 = R.rand(nm)
    m0[::97] = 0.5
    m0[1::97] = 0.0
    m0[2::97] = 1.0
    m0[3::1009] = NAN
    errs, cases = [], [("in range", None, None, [0, 0]), ("image 1.5 at its last element", ni - 1, None, [1, 0]),
                       ("mask -0.25 at its last element", None, nm - 1, [0, 1])]
    for what, bad_i, bad_m, want in cases:
        runs = []
        for _ in range(2 if bad_i is None and bad_m is None else 1):
            im = image_flat.clone()
            if bad_i is not None:
                im[bad_i] = 1.5
            mflat, m = flat_buf(R, nm, torch.float32, fill=0.3)  # must stay 0.3: the in-place binarisation stops at n_mask
            m.copy_(m0)
            if bad_m is not None:
                m[bad_m] = -0.25
            flags = torch.zeros(2, dtype=torch.int32, device=R.dev)
            lib.call("ladi_check_binarise", C.c_void_p(im.data_ptr()), ni, C.c_void_p(m.data_ptr()), nm, C.c_void_p(flags.data_ptr()), R.stream)
            runs.append(dict(m=mflat, flags=flags, src=m0 if bad_m is None else torch.where(torch.arange(nm, device=R.dev) == bad_m, -0.25, m0)))
        torch.cuda.synchronize()
        r = runs[0]
        if r["flags"].tolist() != want:
            errs.append(f"{what}: flags {r['flags'].tolist()}, expected {want}")
        if not bool((r["m"][nm:] == 0.3).all()):
            errs.append(f"{what}: mask written past n_mask")
        src = r["src"]
        ref = torch.where(src < 0.5, 0.0, torch.where(src >= 0.5, 1.0, src))
        e, _ = exact(r["m"][:nm], ref, f"{what}: mask")
        errs += e
        if len(runs) == 2:
            errs += determinism(runs, ["m", "flags"])
    return errs, (0.0 if not errs else float("inf"), "bit-exact mask and flags" if not errs else errs[0])


def replay_posterior_sample(R, f, logvar=None):
    """logvar: [rows, cz] values in place of the random ones (past both clamps); NaN must come out NaN, as torch.clamp keeps it."""
    from ladi_vton_b200 import lib
    mp, n, cz, h, w, scale = f["mp"], f["n"], f["cz"], f["h"], f["w"], f["scale"]
    rows = n * h * w
    lv0 = R.rand(rows, cz) * 60 - 36 if logvar is None else logvar
    mom = R.poisoned(rows, mp, torch.cat([R.randn(rows, cz) * 3, lv0], dim=1), dtype=torch.float32)  # logvar past both clamps
    noise = R.randn(n, cz, h, w)
    cnt = n * cz * h * w

    def fresh():
        flat, o = flat_buf(R, cnt, torch.float32)
        return dict(flat=flat, out=o)
    runs = twice(lambda b: lib.call("ladi_posterior_sample", C.c_void_p(mom.data_ptr()), mp, C.c_void_p(noise.data_ptr()), n, cz, h, w, scale,
                                     C.c_void_p(b["out"].data_ptr()), R.stream), fresh)
    errs = tail_nan(runs[0]["flat"], cnt, "output") + determinism(runs, ["flat"])
    m4 = mom.view(n, h, w, mp).permute(0, 3, 1, 2).double()
    mean, lv = m4[:, :cz], m4[:, cz:2 * cz].clamp(-30.0, 20.0)
    sn = torch.exp(0.5 * lv) * noise.double()
    r = (mean + sn) * scale
    bound = abs(scale) * (2.0 ** -23 * mean.abs() + (2.0 ** -22 + 2.0 ** -23) * sn.abs()) + 2.0 ** -23 * r.abs()
    y = runs[0]["out"].view(n, cz, h, w)
    nan = torch.isnan(r)
    if not torch.equal(torch.isnan(y), nan):
        errs.append(f"NaN at {int(torch.isnan(y).sum())} outputs where the reference has {int(nan.sum())} (a NaN logvar must stay NaN)")
    e, res = worst_at(ratio(y.masked_fill(nan, 0.0), r.masked_fill(nan, 0.0), bound.masked_fill(nan, 1.0)), ("image", "channel", "y", "x"))
    return errs + e, res


def _ddim_coefs(R, steps=3):
    ab = torch.tensor([0.01, 0.02, 0.03, 0.05, 0.3, 0.7, 0.95], dtype=torch.float64)[-(steps + 1):]  # alphas-cumprod, noisy to clean
    rows = torch.zeros((steps, 8), dtype=torch.float64)
    rows[:, 0], rows[:, 1] = ab[:steps].rsqrt(), (1 - ab[:steps]).sqrt()
    rows[:, 2], rows[:, 3], rows[:, 4] = ab[1:steps + 1].sqrt(), (1 - ab[1:steps + 1] - 0.01).sqrt(), 0.1
    return rows.float().to(R.dev)


def replay_ddim_cfg_step(R, f, start=0):
    """Three consecutive calls from device step index `start`: with advance, rows start, start + 1, start + 2 of the coefficient table
    and step_ptr = [s + 1, 0] after each; without, row `start` every time and step_ptr untouched."""
    from ladi_vton_b200 import lib
    ep, inp, B, h, w, cfg, g, adv = f["ep"], f["inp"], f["B"], f["h"], f["w"], f["cfg"], f["guidance"], f["advance"]
    assert f["coef"] and f["step"], "the pipeline's DDIM update reads the step counter"
    hw, Bp = h * w, (2 * B if cfg else B)
    eu = R.randn(B * hw, 4)
    eps = torch.cat([eu, eu + 0.3 * R.randn(B * hw, 4)]) if cfg else eu  # conditional = unconditional + a smaller difference
    eps = R.poisoned(Bp * hw, ep, eps, dtype=torch.float32)
    x_init = R.randn(B, 4, h, w)
    uin_init = R.randn(Bp * hw, inp).bfloat16()
    uin_init[:, :4] = NAN
    coef = _ddim_coefs(R, start + 3)
    noise = R.randn(B, 4, h, w) if f["noise"] else None
    g32 = float(np.float32(g))

    def run(check):
        lat, uin = x_init.clone(), uin_init.clone()
        step = torch.tensor([start, 0], dtype=torch.int32, device=R.dev)
        errs, worst = [], (0.0, "")
        for k in range(3):
            s = start + k if adv else start
            x_before = lat.clone()
            lib.call("ladi_ddim_cfg_step", ptr(eps), ep, ptr(lat), ptr(uin), inp, B, h, w, cfg, g, ptr(coef), ptr(step), adv, ptr(noise), R.stream)
            torch.cuda.synchronize()
            if not check:
                continue
            want_step = [s + 1, 0] if adv else [start, 0]
            if step.tolist() != want_step:
                errs.append(f"step {s}: step_ptr {step.tolist()}, expected {want_step} (grid-wide ticket over {-(-B * 4 * hw // 256)} CTAs)")
            e3 = eps[:, :4].double().view(Bp, h, w, 4).permute(0, 3, 1, 2)
            r, bound = ddim_expect(x_before.double(), e3[:B], e3[B:] if cfg else None, coef[s].double(), g32, cfg,
                                   noise.double() if noise is not None else None)
            q = ratio(lat, r, bound)
            e, res = worst_at(q, ("image", "channel", "y", "x"), f" (step {s}; CTA {int(q.argmax()) // 256})")
            errs += e
            if res[0] > worst[0]:
                worst = res
            want = lat.permute(0, 2, 3, 1).reshape(B * hw, 4).bfloat16()
            u = uin.view(Bp * hw, inp)
            for half in range(Bp // B):
                ee, _ = exact(u[half * B * hw:(half + 1) * B * hw, :4].contiguous(), want, f"step {s}: unet_in rows of CFG half {half}")
                errs += ee
            if not same(u[:, 4:].contiguous(), uin_init[:, 4:].contiguous()):
                errs.append(f"step {s}: unet_in channels >= 4 changed")
        return errs, worst, lat, uin, step
    errs, worst, *first = run(True)
    second = run(False)[2:]
    if not all(same(a, b) for a, b in zip(first, second)):
        errs.append("two runs differ bitwise")
    return errs, worst


def _image_out_input(R, n, h, w, xp):
    v = R.rand(n * h * w, 3) * 2.4 - 1.2  # past both clamps
    k = torch.randint(0, 255, (n * h * w, 3), device=R.dev, generator=R.g).float()
    tie = (k + 0.5) / 127.5 - 1.0  # values whose (x/2 + 0.5) * 255 lands near a rounding tie
    v = torch.where(R.rand(n * h * w, 3) < 0.2, tie, v)
    return R.poisoned(n * h * w, xp, v, dtype=torch.float32)


def replay_image_out(R, f, u8=False, values=None):
    """values: [n*h*w, 3] fp32 in place of the random ones.  NaN: image_out keeps it (torch.clamp); image_out_u8 writes 0."""
    from ladi_vton_b200 import lib
    n, h, w, xp, f32 = f["n"], f["h"], f["w"], f["xp"], f["f32"]
    x = _image_out_input(R, n, h, w, xp) if values is None else R.poisoned(n * h * w, xp, values, dtype=torch.float32)
    if not f32:
        x = x.bfloat16()
    cnt = n * h * w * 3
    dt = torch.uint8 if u8 else torch.float32

    def fresh():
        flat, o = flat_buf(R, cnt, dt, fill=171 if u8 else NAN)
        return dict(flat=flat, out=o)
    name = "ladi_image_out_u8" if u8 else "ladi_image_out"
    runs = twice(lambda b: lib.call(name, C.c_void_p(x.data_ptr()), f32, n, h, w, xp, C.c_void_p(b["out"].data_ptr()), R.stream), fresh)
    tail = runs[0]["flat"][cnt:]
    errs = ([] if bool((tail == 171).all() if u8 else torch.isnan(tail).all()) else ["output: wrote past its end"]) + determinism(runs, ["flat"])
    c = (x[:, :3].float() * 0.5 + 0.5).clamp(0.0, 1.0)
    if u8:
        v = np.rint(c.cpu().numpy() * np.float32(255.0))  # numpy: round half to even
        ref = torch.from_numpy(np.where(np.isnan(v), 0.0, v).astype(np.uint8)).to(R.dev)
    else:
        ref = c
    e, res = exact(runs[0]["out"].view(n * h * w, 3), ref.contiguous(), "values")
    return errs + e, res


def replay_resize_aa(R, f):
    from ladi_vton_b200 import lib
    n, c, h, w, oh, ow, op, c_off = (f[k] for k in ("n", "c", "h", "w", "oh", "ow", "op", "c_off"))
    x = _image(R, n, c, h, w)
    rows = n * oh * ow

    def fresh():
        flat, o = flat_buf(R, rows * op, torch.bfloat16)
        return dict(flat=flat, out=o)
    runs = twice(lambda b: lib.call("ladi_resize_aa", C.c_void_p(x.data_ptr()), n, c, h, w, oh, ow, C.c_void_p(b["out"].data_ptr()), op, c_off, R.stream),
                  fresh)
    out = runs[0]["out"].view(rows, op)
    errs = layout(out, c_off, c_off + c, "output") + tail_nan(runs[0]["flat"], rows * op, "output") + determinism(runs, ["flat"])
    if (oh, ow) == (h, w):  # one tap of weight exactly 1 per output: bf16(x) bit for bit
        errs += exact(out[:, c_off:c_off + c].contiguous(), x.permute(0, 2, 3, 1).reshape(rows, c).bfloat16(), "identity resize")[0]
    worst = (0.0, "")
    for b in pick(n, n * c * h * w, 1 << 24):
        r, bound = resample_expect(x[b].double(), oh, ow, U_BF16)
        e, res = worst_at(ratio(out.view(n, oh, ow, op)[b, ..., c_off:c_off + c].permute(2, 0, 1), r, bound), ("channel", "y", "x"), f" of image {b}")
        errs += e
        worst = max(worst, res)
    return errs, worst


def replay_clip_preprocess(R, f):
    from ladi_vton_b200 import lib
    from ladi_vton_b200.inference import CLIP_MEAN, CLIP_STD
    n, c, h, w, oh, ow, qz = (f[k] for k in ("n", "c", "h", "w", "oh", "ow", "quantise"))
    x = _image(R, n, c, h, w)
    mean, std = torch.tensor(CLIP_MEAN, device=R.dev), torch.tensor(CLIP_STD, device=R.dev)
    cnt = n * c * oh * ow

    def fresh():
        flat, o = flat_buf(R, cnt, torch.float32)
        return dict(flat=flat, out=o)
    runs = twice(lambda b: lib.call("ladi_clip_preprocess", C.c_void_p(x.data_ptr()), n, c, h, w, oh, ow, C.c_void_p(mean.data_ptr()),
                                     C.c_void_p(std.data_ptr()), qz, C.c_void_p(b["out"].data_ptr()), R.stream), fresh)
    errs = tail_nan(runs[0]["flat"], cnt, "output") + determinism(runs, ["flat"])
    y = runs[0]["out"].view(n, c, oh, ow).double()
    md, sd = mean.double().view(c, 1, 1), std.double().view(c, 1, 1)
    worst = (0.0, "")
    for b in pick(n, n * c * h * w, 1 << 24):
        acc, eacc = resample_expect(x[b].double(), oh, ow, 0.0)
        v = (0.5 * acc + 0.5).clamp(0.0, 1.0)
        ev = 0.5 * eacc + 2.0 ** -24
        if qz:  # every level floor(255 v') with |v' - v| within the bound is a correct result
            e255 = 255.0 * ev + 255.0 * EPS24
            lo, hi = torch.floor(255.0 * v - e255), torch.floor(255.0 * v + e255)
            d = torch.full_like(v, float("inf"))
            bnd = torch.ones_like(v)
            for k in range(int((hi - lo).max()) + 1):
                lvl = ((lo + k).clamp_max(hi) / 255.0)
                rk = (lvl - md) / sd
                bk = 2.0 ** -21 * (lvl + md.abs()) / sd + 2.0 ** -24 * rk.abs()
                better = (y[b] - rk).abs() / bk < d / bnd
                d, bnd = torch.where(better, (y[b] - rk).abs(), d), torch.where(better, bk, bnd)
            q = torch.nan_to_num(d / bnd, nan=float("inf"))
        else:
            r = (v - md) / sd
            q = ratio(y[b], r, (ev + 2.0 ** -23 * (v + md.abs())) / sd + U_F32 * r.abs())
        e, res = worst_at(q, ("channel", "y", "x"), f" of image {b}")
        errs += e
        worst = max(worst, res)
    return errs, worst


def _smooth_grid(R, n, gh, gw):
    """A TPS-like sampling grid: the identity lattice, a smooth displacement and a margin that reaches past +-1 (border clipping)."""
    ys, xs = torch.meshgrid(torch.linspace(-1.06, 1.06, gh, device=R.dev), torch.linspace(-1.06, 1.06, gw, device=R.dev), indexing="ij")
    a = R.randn(n, 2, 1, 1) * 0.05
    dx = a[:, 0] * torch.sin(3 * ys + 1)[None] + 0.01 * R.randn(n, gh, gw)
    dy = a[:, 1] * torch.cos(2 * xs)[None] + 0.01 * R.randn(n, gh, gw)
    return torch.stack([xs[None] + dx, ys[None] + dy], dim=3).contiguous()


def replay_warp_grid_sample(R, f, grid=None):
    """grid: fp32 [n, gh, gw, 2] in place of the smooth TPS-like one."""
    from ladi_vton_b200 import lib
    gh, gw, n, c, H, W, op, c_off = (f[k] for k in ("gh", "gw", "n", "c", "H", "W", "op", "c_off"))
    grid = _smooth_grid(R, n, gh, gw) if grid is None else grid.contiguous()
    cloth = _image(R, n, c, H, W)
    rows = n * H * W

    def fresh():
        flat, o = flat_buf(R, rows * op, torch.bfloat16)
        return dict(flat=flat, out=o)
    runs = twice(lambda b: lib.call("ladi_warp_grid_sample", C.c_void_p(grid.data_ptr()), gh, gw, C.c_void_p(cloth.data_ptr()), n, c, H, W,
                                     C.c_void_p(b["out"].data_ptr()), op, c_off, R.stream), fresh)
    out = runs[0]["out"].view(rows, op)
    errs = layout(out, c_off, c_off + c, "output") + tail_nan(runs[0]["flat"], rows * op, "output") + determinism(runs, ["flat"])
    worst = (0.0, "")
    for b in pick(n, n * c * H * W, 1 << 22):
        r, bound = warp_expect(grid[b:b + 1].double(), cloth[b:b + 1].double())
        e, res = worst_at(ratio(out.view(n, H, W, op)[b:b + 1, ..., c_off:c_off + c].permute(0, 3, 1, 2), r, bound), ("", "channel", "y", "x"),
                        f" of image {b}")
        errs += e
        worst = max(worst, res)
    return errs, worst


def relu_features(R, rows, c):
    """post-ReLU activations: half zeros, the rest |N(0, 1)| with per-channel scales."""
    return (R.randn(rows, c).clamp_min(0) * torch.exp(R.randn(c, std=0.5))).bfloat16()


def replay_upsample2x_ac(R, f):
    from ladi_vton_b200 import lib
    n, h, w, c = f["n"], f["h"], f["w"], f["c"]
    x = relu_features(R, n * h * w, c)
    cnt = n * 4 * h * w * c

    def fresh():
        flat, o = flat_buf(R, cnt, torch.bfloat16)
        return dict(flat=flat, out=o)
    runs = twice(lambda b: lib.call("ladi_upsample2x_bilinear_ac", C.c_void_p(x.data_ptr()), n, h, w, c, C.c_void_p(b["out"].data_ptr()), R.stream), fresh)
    errs = tail_nan(runs[0]["flat"], cnt, "output") + determinism(runs, ["flat"])
    worst = (0.0, "")
    for b in pick(n, cnt, 1 << 26):
        r, bound = upsample_ac_expect(x.view(n, h, w, c)[b:b + 1].double())
        e, res = worst_at(ratio(runs[0]["out"].view(n, 2 * h, 2 * w, c)[b:b + 1], r, bound), ("", "y", "x", "channel"), f" of image {b}")
        errs += e
        worst = max(worst, res)
    return errs, worst


def replay_space_to_depth2(R, f):
    from ladi_vton_b200 import lib
    n, h, w, c, xp, op = f["n"], f["h"], f["w"], f["c"], f["xp"], f["op"]
    x = R.poisoned(n * h * w, xp, relu_features(R, n * h * w, c))
    rows = n * (h // 2) * (w // 2)

    def fresh():
        flat, o = flat_buf(R, rows * op, torch.bfloat16)
        return dict(flat=flat, out=o)
    runs = twice(lambda b: lib.call("ladi_space_to_depth2", C.c_void_p(x.data_ptr()), n, h, w, c, xp, C.c_void_p(b["out"].data_ptr()), op, R.stream), fresh)
    out = runs[0]["out"].view(rows, op)
    errs = layout(out, 0, 4 * c, "output") + tail_nan(runs[0]["flat"], rows * op, "output") + determinism(runs, ["flat"])
    ref = x[:, :c].reshape(n, h // 2, 2, w // 2, 2, c).permute(0, 1, 3, 2, 4, 5).reshape(rows, 4 * c)  # channel (sy * 2 + sx) * c + ch
    e, res = exact(out[:, :4 * c].contiguous(), ref.contiguous(), "values")
    return errs + e, res


def replay_maxpool2(R, f, values=None):
    """values: bf16 [n*h*w, c] in place of the post-ReLU features; a window holding a NaN gives NaN, as nn.MaxPool2d does."""
    from ladi_vton_b200 import lib
    n, h, w, c = f["n"], f["h"], f["w"], f["c"]
    x = relu_features(R, n * h * w, c) if values is None else values.bfloat16().contiguous()
    cnt = n * (h // 2) * (w // 2) * c

    def fresh():
        flat, o = flat_buf(R, cnt, torch.bfloat16)
        return dict(flat=flat, out=o)
    runs = twice(lambda b: lib.call("ladi_maxpool2_nhwc", C.c_void_p(x.data_ptr()), n, h, w, c, C.c_void_p(b["out"].data_ptr()), R.stream), fresh)
    errs = tail_nan(runs[0]["flat"], cnt, "output") + determinism(runs, ["flat"])
    ref = F.max_pool2d(x.view(n, h, w, c).permute(0, 3, 1, 2).float(), 2).permute(0, 2, 3, 1).bfloat16().reshape(-1)
    e, res = exact(runs[0]["out"], ref.contiguous(), "values")
    return errs + e, res


def replay_patchify(R, f):
    from ladi_vton_b200 import lib
    n, ch, h, w, ps, kpad = f["n"], f["ch"], f["h"], f["w"], f["patch"], f["kpad"]
    px = R.randn(n, ch, h, w) * 1.2
    rows = n * (h // ps) * (w // ps)

    def fresh():
        flat, o = flat_buf(R, rows * kpad, torch.bfloat16)
        return dict(flat=flat, out=o)
    runs = twice(lambda b: lib.call("ladi_patchify", C.c_void_p(px.data_ptr()), C.c_void_p(b["out"].data_ptr()), n, ch, h, w, ps, kpad, R.stream), fresh)
    errs = tail_nan(runs[0]["flat"], rows * kpad, "output") + determinism(runs, ["flat"])
    ref = torch.zeros((rows, kpad), device=R.dev)
    ref[:, :ch * ps * ps] = F.unfold(px, ps, stride=ps).transpose(1, 2).reshape(rows, -1)  # column (c * ps + ky) * ps + kx
    e, res = exact(runs[0]["out"].view(rows, kpad), ref.bfloat16(), "values (zeros in the padding columns)")
    return errs + e, res


def _sum_round1(y, a, b, names):
    r = a.double() + b.double()
    return worst_at(ratio(y, r, ROUND1 * r.abs()), names)


def replay_vit_assemble(R, f):
    from ladi_vton_b200 import lib
    pp, n, np_, c = f["pp"], f["n"], f["np"], f["c"]
    patch = R.poisoned(n * np_, pp, R.randn(n * np_, c))
    cls, pos = R.randn(c).bfloat16(), (R.randn(np_ + 1, c) * 0.3).bfloat16()
    cnt = n * (np_ + 1) * c

    def fresh():
        flat, o = flat_buf(R, cnt, torch.bfloat16)
        return dict(flat=flat, out=o)
    runs = twice(lambda b: lib.call("ladi_vit_assemble", C.c_void_p(patch.data_ptr()), pp, C.c_void_p(cls.data_ptr()), C.c_void_p(pos.data_ptr()),
                                     C.c_void_p(b["out"].data_ptr()), n, np_, c, R.stream), fresh)
    errs = tail_nan(runs[0]["flat"], cnt, "output") + determinism(runs, ["flat"])
    a = torch.cat([cls.view(1, 1, c).expand(n, 1, c), patch[:, :c].view(n, np_, c)], dim=1)
    e, res = _sum_round1(runs[0]["out"].view(n, np_ + 1, c), a, pos.view(1, np_ + 1, c), ("image", "token", "channel"))
    return errs + e, res


def replay_clip_embed(R, f):
    from ladi_vton_b200 import lib
    rows, seq, c, op = f["rows"], f["seq"], f["c"], f["op"]
    B, V, nv = rows // seq, 49408, 16
    tok, pos = (R.randn(V, c) * 0.02).bfloat16(), (R.randn(seq, c) * 0.01).bfloat16()
    src = torch.randint(0, V, (B, seq), device=R.dev, generator=R.g, dtype=torch.int32)
    wemb = None
    if f["wemb"]:
        wemb = R.randn(B * nv, c).bfloat16()
        for b in range(B):  # the pseudo-words of prompt b start at a different token of each prompt, up to the last position
            s0 = seq - nv - (b * 7) % (seq - nv)
            src[b, s0:s0 + nv] = -(b * nv + torch.arange(nv, device=R.dev, dtype=torch.int32)) - 1
    src = src.view(-1).contiguous()

    def fresh():
        flat, o = flat_buf(R, rows * op, torch.bfloat16)
        return dict(flat=flat, out=o)
    runs = twice(lambda b: lib.call("ladi_clip_embed", ptr(src), ptr(tok), ptr(wemb), ptr(pos), ptr(b["out"]), rows, seq, c, op, R.stream), fresh)
    out = runs[0]["out"].view(rows, op)
    errs = layout(out, 0, c, "output") + tail_nan(runs[0]["flat"], rows * op, "output") + determinism(runs, ["flat"])
    sl = src.long()
    e = tok[sl.clamp_min(0)]
    if wemb is not None:
        e = torch.where((sl < 0)[:, None], wemb[(-sl - 1).clamp(0, B * nv - 1)], e)
    ee, res = _sum_round1(out[:, :c], e, pos[torch.arange(rows, device=R.dev) % seq], ("row", "channel"))
    return errs + ee, res


def replay_channel_affine(R, f):
    from ladi_vton_b200 import lib
    rows, c, pitch = f["rows"], f["c"], f["pitch"]
    x0 = R.poisoned(rows, pitch, relu_features(R, rows, c))
    s, t = (R.rand(c) + 0.5) / (R.rand(c) + 0.5).sqrt(), R.randn(c) * 0.3

    def fresh():
        return dict(x=x0.clone())
    runs = twice(lambda b: lib.call("ladi_channel_affine", C.c_void_p(b["x"].data_ptr()), rows, c, pitch, C.c_void_p(s.data_ptr()), C.c_void_p(t.data_ptr()),
                                     R.stream), fresh)
    errs = layout(runs[0]["x"], 0, c, "in-place output") + determinism(runs, ["x"])
    r = x0[:, :c].double() * s.double() + t.double()
    e, res = worst_at(ratio(runs[0]["x"][:, :c], r, (U_BF16 + EPS24) * r.abs()), ("row", "channel"))
    return errs + e, res


def replay_l2norm_channels(R, f, values=None):
    from ladi_vton_b200 import lib
    rows, c, pitch = f["rows"], f["c"], f["pitch"]
    x0 = R.poisoned(rows, pitch, relu_features(R, rows, c) if values is None else values)

    def fresh():
        return dict(x=x0.clone())
    runs = twice(lambda b: lib.call("ladi_l2norm_channels", C.c_void_p(b["x"].data_ptr()), rows, c, pitch, R.stream), fresh)
    errs = layout(runs[0]["x"], 0, c, "in-place output") + determinism(runs, ["x"])
    xd = x0[:, :c].double()
    r = xd / torch.sqrt((xd * xd).sum(1, keepdim=True) + 1e-6)
    e, res = worst_at(ratio(runs[0]["x"][:, :c], r, (U_BF16 + 0.5 * C_ACC * math.sqrt(c) * EPS24 + 2.0 ** -22) * r.abs()), ("row", "channel"))
    return errs + e, res


def replay_feature_correlation(R, f):
    from ladi_vton_b200 import lib
    n, h, w, c, op = f["n"], f["h"], f["w"], f["c"], f["op"]
    hw = h * w

    def unit(rows):  # FeatureL2Norm outputs: post-ReLU features scaled to unit length per pixel
        a = relu_features(R, rows, c).float()
        return (a / a.norm(dim=1, keepdim=True).clamp_min(1e-3)).bfloat16()
    fa, fb = unit(n * hw), unit(n * hw)

    def fresh():
        flat, o = flat_buf(R, n * hw * op, torch.bfloat16)
        return dict(flat=flat, out=o)
    runs = twice(lambda b: lib.call("ladi_feature_correlation", C.c_void_p(fa.data_ptr()), C.c_void_p(fb.data_ptr()), n, h, w, c,
                                     C.c_void_p(b["out"].data_ptr()), op, R.stream), fresh)
    out = runs[0]["out"].view(n * hw, op)
    errs = layout(out, 0, hw, "output") + tail_nan(runs[0]["flat"], n * hw * op, "output") + determinism(runs, ["flat"])
    r, bound = corr_expect(fa.view(n, h, w, c).double(), fb.view(n, h, w, c).double())
    e, res = worst_at(ratio(out.view(n, h, w, op)[..., :hw], r, bound), ("image", "yB", "xB", "channel xA*h+yA"))
    return errs + e, res


def tps_expect(theta, inv, rep, n_ctrl):
    """theta [n, 2 n_ctrl], inv [K, K], rep [P, K] float64 (K = n_ctrl + 3) -> (points, points bound, grid, grid bound)."""
    n = theta.shape[0]
    pts = torch.tanh(theta).view(n, n_ctrl, 2)
    ep = 2.0 ** -22 * pts.abs()
    mapping = inv[:, :n_ctrl] @ pts  # [n, K, 2]: the 3 padding rows of the control-point matrix are zero
    em = inv[:, :n_ctrl].abs() @ (ep + C_ACC * math.sqrt(n_ctrl) * EPS24 * pts.abs())
    grid = rep @ mapping
    K = rep.shape[1]
    eg = rep.abs() @ em + C_ACC * math.sqrt(K) * EPS24 * (rep.abs() @ mapping.abs())
    return pts, ep + 2.0 ** -126, grid, eg + EPS24 * grid.abs()


def replay_tps_grid(R, f):
    from ladi_vton_b200 import lib
    from ladi_vton_b200.warp import control_points, tps_matrices
    tp, n, nc, npts = f["tp"], f["n"], f["n_ctrl"], f["npts"]
    if (nc, npts) == (25, 256 * 192):  # the ConvNet_TPS(256, 192) matrices
        inv, rep = (t.to(R.dev).contiguous() for t in tps_matrices(256, 192, control_points()))
        theta = R.poisoned(n, tp, torch.atanh(control_points().to(R.dev)).view(1, -1) + 0.2 * R.randn(n, 2 * nc), dtype=torch.float32)
    else:  # other control-point and pixel counts: matrices of the same magnitudes
        K = nc + 3
        inv, rep = R.randn(K, K) * 2, torch.cat([R.rand(npts, K - 2) * 2 - 1, R.rand(npts, 2) * 2 - 1], dim=1)
        theta = R.poisoned(n, tp, R.randn(n, 2 * nc), dtype=torch.float32)

    def fresh():
        pf, p = flat_buf(R, n * nc * 2, torch.float32)
        gf, g = flat_buf(R, n * npts * 2, torch.float32)
        return dict(pf=pf, p=p, gf=gf, g=g)
    runs = twice(lambda b: lib.call("ladi_tps_grid", C.c_void_p(theta.data_ptr()), tp, C.c_void_p(inv.data_ptr()), C.c_void_p(rep.data_ptr()), n, nc, npts,
                                     C.c_void_p(b["p"].data_ptr()), C.c_void_p(b["g"].data_ptr()), R.stream), fresh)
    errs = (tail_nan(runs[0]["pf"], n * nc * 2, "points") + tail_nan(runs[0]["gf"], n * npts * 2, "grid") + determinism(runs, ["pf", "gf"]))
    pts, bp, grid, bg = tps_expect(theta[:, :2 * nc].double(), inv.double(), rep.double(), nc)
    e1, r1 = worst_at(ratio(runs[0]["p"].view(n, nc, 2), pts, bp), ("image", "control point", "coordinate"), " (points)")
    e2, r2 = worst_at(ratio(runs[0]["g"].view(n, npts, 2), grid, bg), ("image", "pixel", "coordinate"), " (grid)")
    return errs + e1 + e2, max(r1, r2)


def replay_attention_small(R, f):
    B, heads, nq, nkv, hd = (f[k] for k in ("B", "heads", "nq", "nkv", "hd"))
    Cw = heads * hd
    bufs = {}
    for nm, n_, std in (("q", nq, 2 ** 0.5), ("k", nkv, 2 ** 0.5), ("v", nkv, 1.0)):
        p, bs = f[nm + "p"], f[nm + "bs"]
        t = torch.full(((B - 1) * bs + n_ * p,), NAN, dtype=torch.bfloat16, device=R.dev)
        t.as_strided((B, n_, Cw), (bs, p, 1)).copy_(R.randn(B, n_, Cw, std=std).bfloat16())
        bufs[nm] = t
    return check_attention_small(R, f, bufs)


def check_attention_small(R, f, bufs):
    """Run the descriptor f twice on the inputs bufs["q" / "k" / "v"] (bf16 tensors whose storage offset is the operand's address; they
    may be views into one buffer) into a NaN-poisoned output with a tail, then check the layout, determinism and the float64 bound of
    every query row of every image."""
    from ladi_vton_b200 import lib
    B, heads, nq, nkv, hd, causal, scale = (f[k] for k in ("B", "heads", "nq", "nkv", "hd", "causal", "scale"))
    Cw = heads * hd
    op, obs = f["op"], f["obs"]
    size = (B - 1) * obs + nq * op

    def fresh():
        flat, o = flat_buf(R, size, torch.bfloat16)
        return dict(flat=flat, out=o)
    runs = twice(lambda b: lib.call("ladi_attention_small", ptr(bufs["q"]), ptr(bufs["k"]), ptr(bufs["v"]), ptr(b["out"]), B, heads, nq, nkv, hd,
                                     f["qp"], f["kp"], f["vp"], op, f["qbs"], f["kbs"], f["vbs"], obs, scale, causal, R.stream), fresh)
    flat = runs[0]["flat"]
    ov = flat.as_strided((B, nq, Cw), (obs, op, 1))
    owned = torch.zeros(flat.numel(), dtype=torch.bool, device=R.dev)  # every element of the flat buffer: row padding, gaps between images, tail
    owned.as_strided((B, nq, Cw), (obs, op, 1)).fill_(True)
    errs = determinism(runs, ["flat"])
    fl = flat.float()
    if not bool(torch.isfinite(fl[owned]).all()):
        errs.append(f"output: non-finite at flat element {int((owned & ~torch.isfinite(fl)).nonzero()[0])} of the B x nq x heads*hd it owns")
    if not bool(torch.isnan(fl[~owned]).all()):
        errs.append(f"output: wrote flat element {int((~owned & ~torch.isnan(fl)).nonzero()[0])}, outside the rows and columns it owns")
    worst = (0.0, "")
    for b in range(B):  # every image and every query row: a causal off-by-one shows in the rows it shifts
        q, k, v = (bufs[nm].as_strided((B, n_, Cw), (f[nm + "bs"], f[nm + "p"], 1))[b].double() for nm, n_ in (("q", nq), ("k", nkv), ("v", nkv)))
        o, bound = small_attn_expect(q, k, v, heads, scale, causal)
        qq = ratio(ov[b], o, bound).view(nq, heads, hd)
        e, res = worst_at(qq, ("query", "head", "column"), f" of image {b}")
        errs += e
        worst = max(worst, res)
    return errs, worst


REPLAY = {"conv": replay_conv, "ln": replay_ln, "check_binarise": replay_check_binarise, "bilinear_down8": replay_bilinear_down8,
          "nchw_to_nhwc": replay_nchw_to_nhwc, "posterior_sample": replay_posterior_sample, "inv_mask_rows": replay_inv_mask_rows,
          "ddim_cfg_step": replay_ddim_cfg_step, "image_out": replay_image_out,
          "image_out_u8": functools.partial(replay_image_out, u8=True), "resize_aa": replay_resize_aa,
          "clip_preprocess": replay_clip_preprocess, "space_to_depth2": replay_space_to_depth2, "channel_affine": replay_channel_affine,
          "l2norm_channels": replay_l2norm_channels, "feature_correlation": replay_feature_correlation, "tps_grid": replay_tps_grid,
          "warp_grid_sample": replay_warp_grid_sample, "maxpool2": replay_maxpool2, "upsample2x_ac": replay_upsample2x_ac,
          "nhwc_to_nchw_clamp": replay_nhwc_to_nchw_clamp, "attention_small": replay_attention_small, "clip_embed": replay_clip_embed,
          "patchify": replay_patchify, "vit_assemble": replay_vit_assemble}
