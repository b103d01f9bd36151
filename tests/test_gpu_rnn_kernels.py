"""`pytest -m gpu`: the recurrent kernels of GRU and LSTM (rnn.cu rnn_cluster_kernel, rnn_step_gates_kernel and
rnn_state_init_kernel), each selected by name and checked bit for bit.

The launchers pick the cluster kernel's instance, cluster size, batch slice and shared memory from H, B, the direction
count and the SM count, or the per-step path (api_rnn.cu) when R does not fit a 16-CTA cluster.  The rules are restated
below (`cluster_rule`, `per_step_rule`); `VARIANTS` lists every instance they pick from
(tests/test_rnn_kernel_table_cpu.py keeps it equal to the built library's symbols).  `EDGES` lists the branches a kernel
name does not show; the case list reaches each of them, and every instance at least twice, on 132 and on 114 SMs.  The
per-step path's recurrent product runs skinny_f32_kernel, the wgmma GEMM, the 3xTF32 split and the strided copy, which
belong to the tables of tests/test_gpu_row_kernels.py and tests/test_gpu_staging_kernels.py; the rule here names them
but this table does not list them.

  * kernel identity: every case runs once under CUPTI in a child process and must run exactly the RNN instances and
    per-step kernels its rule names, with the grid and 256-thread block the rule gives, and (where Kineto records it)
    the cluster launch's shared memory.  Kineto does not record cluster dimensions: the cluster size C is checked through
    what it determines, the grid of C * dirs * slices CTAs, the BT instance and the shared memory.  A 16-CTA cluster also depends on cudaOccupancyMaxActiveClusters, which no
    rule restates: such a case either runs the cluster kernel on 16 * dirs * slices CTAs or falls back to exactly the
    per-step launches, and the test prints which;
  * values against `rnn_model`, a float32 restatement of the kernels' order of operations.  x and W hold multiples of
    2^-5 in [-1, 1] with I <= 128, so every partial sum of the input projection is a multiple of 2^-10 below 2^7: exact
    in f32 and in TF32, in any order and in both f32 modes.  R, the biases, h0 and c0 are full-mantissa floats, so the
    recurrence is sensitive to every rounding.  The cluster product is one fma chain per output over k = 0 .. Hp - 1,
    the skinny product restates skinny_f32_kernel's lane chains and reduction, the gates follow gate_update one rounded
    operation at a time, and the LSTM's tanhf(c) (libdevice, not restated) comes from `tanhf_probe`.  The per-step wgmma
    product (B > 32) runs in 3xTF32 and is not exact: it is held to `WGMMA_BOUND` against the model with a float64
    product, and must give the same bits on a rerun and from a replayed CUDA graph;
  * R (also as a transposed view), h0, c0 and the bias go in as strided views of buffers filled with NaN, so a finite
    bit-exact result shows nothing outside the views is read.  The cluster kernel reads R through the caller's strides
    (transposed, padded rows, padded directions, an offset base); the per-step path copies such an R to dense rows
    first (the strided copy), or reads 16-byte rows with NaN padding in place."""
import json

import numpy as np
import pytest

import gpu_checks as gc
import test_gpu_conv_norm_resize_kernels as ck
import test_gpu_decode_step_kernels as dk
import test_gpu_row_kernels as rk

pytestmark = pytest.mark.gpu

F32 = np.float32
THREADS = 256
MAX_SMEM = 227 * 1024  # sm_90 opt-in shared memory per block (RNN_MAX_SMEM)
WGMMA_BOUND = 1e-5  # |GPU - model| on Y, Y_h, Y_c when the per-step product runs on the wgmma GEMM (3xTF32)

# ---- the kernels ------------------------------------------------------------------------------------------------------
VARIANTS = {
    "rnn_cluster_kernel": [(g, bt) for g in (1, 0) for bt in (8, 4, 2, 1)],  # <GRU, BT>
    "rnn_step_gates_kernel": [(1,), (0,)],  # <GRU>
    "rnn_state_init_kernel": [()],
}
KERNELS = set(VARIANTS)
# the per-step path's product and staging kernels, named by their own tables
STEP_KERNELS = {"skinny_f32_kernel"}
EDGES = tuple(f"C = {c}" for c in (1, 2, 4, 8, 16)) + (
    "thread clamp", "shared-memory shrink", "Bsp > Bs", "B % Bs != 0", "H % C != 0", "H % 4 != 0", "RS = Hp",
    "RS = Hp + 4", "forward", "reverse", "bidirectional", "no bias", "no h0 / c0", "T = 0", "T = 1", "I = 0",
    "per-step MT 8", "per-step MT 16", "per-step MT 32", "per-step wgmma", "R copied: r_k != 1", "R copied: H % 4 != 0",
    "R copied: row stride", "R copied: direction stride", "R copied: base alignment", "R in place")


def kernel_key(name, kernels=KERNELS):
    return ck.kernel_key(name, kernels)


def _cdiv(a, b):
    return -(-a // b)


def _r4(n):
    return _cdiv(n, 4) * 4


# ---- the cluster rule (rnn.cu plan_cluster / cluster_smem) --------------------------------------------------------------
def cluster_smem(G, C, H, Bsp):
    """(bytes, Hc, Hp, RS): R's rows [G Hc][RS], h double-buffered [2][Bsp][Hp], products [G Hc][Bsp]; RS = Hp, or
    Hp + 4 when Hp / 4 is even, so that RS / 4 is odd"""
    Hc, Hp = _cdiv(H, C), _r4(H)
    rs4 = Hp // 4
    rs4 += rs4 % 2 == 0
    RS = rs4 * 4
    return 4 * (G * Hc * RS + 2 * Bsp * Hp + G * Hc * Bsp), Hc, Hp, RS


def batch_tile(Bs):
    return 8 if Bs >= 8 else 4 if Bs >= 4 else 2 if Bs >= 2 else 1


def cluster_rule(sms, gru, H, B, dirs, min_C=1):
    """plan_cluster: the smallest C >= min_C (a power of two up to 16) whose shared memory holds its G * ceil(H / C) rows
    of R with one batch row and whose units fit the 256 threads; then Bs = ceil(B / slices wanted) with slices wanted =
    max(1, SMs / C / dirs), clamped to 256 / Hc gate threads and lowered until shared memory holds Bsp rows (Bs rounded
    up to BT).  None above the cluster bound."""
    G = 3 if gru else 4
    if H < 1 or B < 1:
        return None
    C = min_C
    while C <= 16:
        smem1, Hc, Hp, RS = cluster_smem(G, C, H, 1)
        if smem1 > MAX_SMEM or Hc > THREADS:
            C *= 2
            continue
        want = max(1, sms // C // dirs)
        wanted = max(1, _cdiv(B, want))
        Bs = min(wanted, THREADS // Hc)
        clamped = Bs
        while Bs > 1:
            bt = batch_tile(Bs)
            if cluster_smem(G, C, H, _cdiv(Bs, bt) * bt)[0] <= MAX_SMEM:
                break
            Bs -= 1
        BT = batch_tile(Bs)
        Bsp = _cdiv(Bs, BT) * BT
        slices = _cdiv(B, Bs)
        return dict(C=C, Hc=Hc, Hp=Hp, RS=RS, Bs=Bs, BT=BT, Bsp=Bsp, slices=slices, smem=cluster_smem(G, C, H, Bsp)[0],
                    grid=C * dirs * slices, block=THREADS, clamp=clamped < wanted, shrink=Bs < clamped)
    return None


# ---- the per-step rule (api_rnn.cu rnn_run, rnn.cu launch_rnn_state_init / launch_rnn_step_gates) ------------------------
def r_layout(layout, dirs, GH, H):
    """(strides, element offset, buffer size) of R's view [dirs, G H, H] in a NaN-filled device buffer, or None: the
    host array as given (dense, copied to a 256-byte aligned device buffer by the call)"""
    if layout == "host":
        return None
    if layout == "T":  # stored [dirs, H, G H + 1]: a transposed view
        return (H * (GH + 1), 1, GH + 1), 0, dirs * H * (GH + 1)
    if layout == "rowpad1":  # rows of H + 1
        return (GH * (H + 1), H + 1, 1), 0, dirs * GH * (H + 1)
    if layout == "rowpad4":  # rows of H + 4, directions 4 apart more: 16-byte rows, used in place
        return (GH * (H + 4) + 4, H + 4, 1), 0, dirs * (GH * (H + 4) + 4)
    if layout == "dirpad":  # dense rows, directions GH H + 2 apart
        return (GH * H + 2, H, 1), 0, dirs * (GH * H + 2)
    if layout == "offset1":  # dense, one element into the buffer
        return (GH * H, H, 1), 1, dirs * GH * H + 1
    raise ValueError(layout)


def r_copy_reasons(layout, dirs, G, H):
    """api_rnn.cu: R is copied into a zero-padded [dirs, G H, round_up(H, 4)] buffer when r_k != 1, H % 4 != 0, the row
    or direction stride is not a multiple of 4, or the base is not 16-byte aligned"""
    GH = G * H
    lay = r_layout(layout, dirs, GH, H)
    (sd, sr, sk), off = lay[:2] if lay else ((GH * H, H, 1), 0)
    why = set()
    if sk != 1:
        why.add("R copied: r_k != 1")
    if H % 4:
        why.add("R copied: H % 4 != 0")
    if sr % 4:
        why.add("R copied: row stride")
    if sd % 4:
        why.add("R copied: direction stride")
    if off % 4:
        why.add("R copied: base alignment")
    return why


def per_step_rule(s, sms):
    """(the launches [(key, grid)], {kernel family: launches} of the product / staging kernels, what the rule saw).
    One state init (grid min(ceil(n / 256), 4 SMs), n = dirs B H), then per step one product per direction and one
    gate launch (grid ceil(n / 256)).  The product: skinny_f32_kernel over K = round_up(H, 4) for B <= 32 (instance and
    grid as rk.skinny_rule and launch_skinny_f32), else the wgmma GEMM forced to 3xTF32, with R split once per
    direction before the first step and h split at every step."""
    op, T, B, I, H, dirs = s["op"], s["T"], s["B"], s["I"], s["H"], _dirs(s)
    G = 3 if op == "gru" else 4
    GH, n = G * H, dirs * B * H
    copied = r_copy_reasons(s.get("r", "host"), dirs, G, H)
    launches = [(("rnn_state_init_kernel", ()), min(_cdiv(n, 256), 4 * sms))]
    product = "skinny" if B <= 32 else "wgmma"
    if product == "skinny":
        key = rk.skinny_rule(B, GH)
        tiles = _cdiv(GH, 8 * key[1][1])
        launches += [(key, min(tiles, 2 * sms))] * (T * dirs)
    launches += [(("rnn_step_gates_kernel", (int(op == "gru"),)), _cdiv(n, 256))] * T
    others = {"umma": T * dirs if product == "wgmma" else 0, "tf32x3": dirs + T * dirs if product == "wgmma" else 0,
              "nd_copy": int(bool(copied))}
    return launches, others, dict(copied=copied, product=product, mt=rk.skinny_rule(B, GH)[1][0] if B <= 32 else None)


def _dirs(s):
    return 2 if s["dir"] == "bidirectional" else 1


def projection_launches(s):
    """the input projection's kernels: one wgmma GEMM when I > 0 (a memset otherwise); in 3xTF32 its two operand splits;
    x and W copied to 16-byte rows when I % 4 != 0"""
    I = s["I"]
    if I == 0 or s["T"] == 0:
        return {"umma": 0, "tf32x3": 0, "nd_copy": 0}
    return {"umma": 1, "tf32x3": 2 if s.get("x3", True) else 0, "nd_copy": 2 if I % 4 else 0}


def case_rule(s, sms):
    """dict(path: "init" (T = 0), "cluster" or "per-step"; plan: the cluster rule (or None); launches / others for the
    per-step path; edges)"""
    op, T, B, I, H, dirs = s["op"], s["T"], s["B"], s["I"], s["H"], _dirs(s)
    gru = op == "gru"
    plan = None if s.get("step") else cluster_rule(sms, gru, H, B, dirs)
    edges = {s["dir"]}
    if not s.get("bias", True):
        edges.add("no bias")
    if not s.get("init", True):
        edges.add("no h0 / c0")
    if T in (0, 1):
        edges.add(f"T = {T}")
    if I == 0:
        edges.add("I = 0")
    if H % 4:
        edges.add("H % 4 != 0")
    if T == 0:
        n = dirs * B * H
        return dict(path="init", plan=None, launches=[(("rnn_state_init_kernel", ()), min(_cdiv(n, 256), 4 * sms))],
                    others={"umma": 0, "tf32x3": 0, "nd_copy": 0}, edges=edges)
    launches, others, seen = per_step_rule(s, sms)
    if plan is not None:
        edges.add(f"C = {plan['C']}")
        edges |= {e for e, on in (("thread clamp", plan["clamp"]), ("shared-memory shrink", plan["shrink"]),
                                  ("Bsp > Bs", plan["Bsp"] > plan["Bs"]), ("B % Bs != 0", B % plan["Bs"] != 0),
                                  ("H % C != 0", H % plan["C"] != 0)) if on}
        edges.add("RS = Hp" if plan["RS"] == plan["Hp"] else "RS = Hp + 4")
    if plan is None or plan["C"] == 16:  # the per-step launches (a 16-CTA cluster may fall back to them)
        edges.add("per-step wgmma" if seen["product"] == "wgmma" else f"per-step MT {seen['mt']}")
        edges |= seen["copied"] or {"R in place"}
    return dict(path="cluster" if plan else "per-step", plan=plan, launches=launches, others=others, edges=edges)


# ---- the cases --------------------------------------------------------------------------------------------------------
def _batch_for(op, H, dirs, bt, sms, ragged=False):
    """the smallest batch whose cluster plan has batch tile `bt` (and, `ragged`, a partial last slice)"""
    for B in range(1, 20000):
        p = cluster_rule(sms, op == "gru", H, B, dirs)
        if p and p["BT"] == bt and (not ragged or B % p["Bs"]):
            return B
    raise AssertionError(f"no batch gives BT = {bt} for {op} H = {H} on {sms} SMs")


def specs(sms):
    c = lambda op, T, B, I, H, d, **kw: dict(op=op, T=T, B=B, I=I, H=H, dir=d, **kw)  # noqa: E731
    bt = lambda op, H, dirs, t, ragged=False: _batch_for(op, H, dirs, t, sms, ragged)  # noqa: E731
    return [
        # GRU on the cluster kernel: every C, the thresholds of C = 2 / 4 / 8 / 16, the clamp, the shrink, the padding
        c("gru", 3, bt("gru", 16, 1, 8), 32, 16, "forward"),
        c("gru", 2, 5000, 4, 1, "forward"),  # BT 8 with Bsp > Bs
        c("gru", 3, bt("gru", 137, 2, 2), 16, 137, "bidirectional", views=True, r="T"),
        c("gru", 4, bt("gru", 195, 1, 4), 8, 195, "reverse", bias=False, r="offset1"),
        c("gru", 3, 1, 128, 277, "forward", init=False),
        c("gru", 2, 3, 20, 389, "bidirectional", r="dirpad"),
        c("gru", 2, 64, 12, 193, "bidirectional", r="rowpad1"),  # the shared-memory shrink: C = 2, Bs = 1
        c("gru", 2, 264, 8, 256, "forward"),  # the thread clamp
        c("gru", 1, 5, 0, 544, "forward"),  # the largest GRU cluster
        c("gru", 0, 3, 8, 10, "bidirectional", init=False),
        c("gru", 3, bt("gru", 40, 1, 2, ragged=True), 24, 40, "reverse", views=True, r="rowpad4"),
        c("gru", 2, 100, 8, 20, "forward", x3=False),
        # LSTM on the cluster kernel
        c("lstm", 3, bt("lstm", 8, 2, 8), 16, 8, "bidirectional", views=True, r="dirpad"),
        c("lstm", 2, bt("lstm", 20, 1, 8, ragged=True), 32, 20, "forward"),
        c("lstm", 3, bt("lstm", 117, 1, 4), 64, 117, "forward", r="rowpad1"),
        c("lstm", 3, bt("lstm", 30, 1, 4), 8, 30, "reverse", bias=False, init=False, r="offset1"),
        c("lstm", 3, bt("lstm", 167, 1, 2), 16, 167, "reverse", bias=False),
        c("lstm", 2, bt("lstm", 64, 2, 2), 4, 64, "bidirectional", views=True, x3=False, r="T"),
        c("lstm", 3, 1, 40, 237, "forward", init=False),
        c("lstm", 2, 5, 12, 337, "bidirectional", r="T"),
        c("lstm", 2, 2, 8, 468, "forward"),  # the largest LSTM cluster
        c("lstm", 0, 4, 8, 12, "forward", views=True),
        c("lstm", 1, 3, 0, 50, "reverse"),
        c("lstm", 3, 100, 8, 24, "forward"),
        # the per-step path: forced (step=True) or above the cluster bound
        c("gru", 3, 8, 16, 64, "forward", step=True),
        c("lstm", 2, 12, 32, 600, "bidirectional", r="T"),
        c("gru", 2, 20, 8, 550, "forward"),
        c("lstm", 3, 40, 16, 36, "bidirectional", step=True),
        c("gru", 2, 48, 64, 600, "reverse"),
        c("lstm", 2, 33, 0, 512, "forward"),
        c("gru", 3, 3, 8, 32, "forward", step=True, r="rowpad1", views=True),
        c("lstm", 2, 5, 8, 16, "bidirectional", step=True, r="dirpad", x3=False),
        c("gru", 2, 16, 12, 24, "reverse", step=True, r="offset1", bias=False),
        c("lstm", 3, 32, 20, 64, "forward", step=True, r="rowpad4", views=True),
        c("gru", 1, 9, 4, 7, "forward", step=True, r="T"),
        c("gru", 2, 2, 8, 1030, "bidirectional"),  # K = 1032: a chunk of 1024 and one of 8 on the skinny kernel
    ]


def spec_id(s):
    return " ".join(f"{k}={v}" for k, v in s.items())


def coverage_gaps(sms):
    """instances that fewer than two cases select (16-CTA cases not counted: they may fall back), and edges no case
    reaches"""
    picked, reached = {}, set()
    for s in specs(sms):
        r = case_rule(s, sms)
        keys = []
        if r["path"] == "cluster":
            keys.append(("rnn_cluster_kernel", (int(s["op"] == "gru"), r["plan"]["BT"])))
        if r["path"] != "cluster":
            keys += [k for k, _ in r["launches"] if k[0] in KERNELS]
        if r["plan"] is None or r["plan"]["C"] < 16:
            for k in set(keys):
                assert k[1] in VARIANTS[k[0]], f"{spec_id(s)}: the rule names {k}, which the table lacks"
                picked[k] = picked.get(k, 0) + 1
        reached |= r["edges"]
    gaps = [("selected fewer than twice", (k, a)) for k, args in VARIANTS.items() for a in args if picked.get((k, a), 0) < 2]
    return gaps + [("edge never reached", e) for e in EDGES if e not in reached]


# ---- inputs -----------------------------------------------------------------------------------------------------------
def _rng(*key):
    return rk._rng("rnn", *key)


def prepare(s):
    """host inputs: x and W multiples of 2^-5 in [-1, 1] (W in [-1/4, 1/4]), R / bias / h0 / c0 full-mantissa floats"""
    op, T, B, I, H, dirs = s["op"], s["T"], s["B"], s["I"], s["H"], _dirs(s)
    G = 3 if op == "gru" else 4
    r = _rng(spec_id(s))
    k = F32(1 / np.sqrt(H))
    inp = dict(x=(r.integers(-32, 33, (T, B, I)) / 32).astype(F32), w=(r.integers(-8, 9, (dirs, G * H, I)) / 32).astype(F32),
               r=r.uniform(-k, k, (dirs, G * H, H)).astype(F32))
    inp["b"] = r.uniform(-k, k, (dirs, 2 * G * H)).astype(F32) if s.get("bias", True) else None
    inp["h0"] = r.uniform(-0.5, 0.5, (dirs, B, H)).astype(F32) if s.get("init", True) else None
    inp["c0"] = r.uniform(-2, 2, (dirs, B, H)).astype(F32) if s.get("init", True) and op == "lstm" else None
    return inp


def _nan_view(ctx, a, strides, off, size):
    """`a` on the device as the view (strides, off) of a buffer of `size` NaNs"""
    buf = np.full(size, np.nan, F32)
    idx = off + sum(np.arange(n).reshape([-1 if i == j else 1 for j in range(a.ndim)]) * st
                    for i, (n, st) in enumerate(zip(a.shape, strides)))
    buf[idx] = a
    return ctx.to_device(buf).view(a.shape, strides, off)


def device_args(ctx, s, inp):
    """the call's arguments: R in its layout, and with `views` h0 / c0 / bias as strided views, all in NaN buffers"""
    dirs, H, B = _dirs(s), s["H"], s["B"]
    GH = inp["r"].shape[1]
    lay = r_layout(s.get("r", "host"), dirs, GH, H)
    args = dict(r=inp["r"] if lay is None else _nan_view(ctx, inp["r"], *lay))
    for name, key in (("b", "b"), ("initial_h", "h0"), ("initial_c", "c0")):
        a = inp[key]
        if a is None:
            continue
        if not s.get("views"):
            args[name] = a
        elif name == "b":  # every second element
            args[name] = _nan_view(ctx, a, (4 * GH, 2), 0, dirs * 4 * GH)
        else:  # rows of H + 3, one element in
            args[name] = _nan_view(ctx, a, (B * (H + 3), H + 3, 1), 1, dirs * B * (H + 3) + 1)
    return args


def run_case(rt, ctx, s, inp, args=None):
    """(Y, Y_h[, Y_c]) as host arrays"""
    args = device_args(ctx, s, inp) if args is None else args
    ctx.set_f32_mode(s.get("x3", True))
    o = rt.GRU(s["dir"], s["H"]) if s["op"] == "gru" else rt.LSTM(s["dir"], s["H"])
    kw = {k: v for k, v in args.items() if k != "r"}
    with gc.switches(RTEN_B200_NO_RNN_CLUSTER=1 if s.get("step") else None):
        out = o.run(ctx, inp["x"], inp["w"], args["r"], **kw)
    return [t.numpy() for t in out]


# ---- the model --------------------------------------------------------------------------------------------------------
def _fma(a, b, c):
    from oracle.norms import fma_f32
    return fma_f32(a, b, c)


def product_chain(h, R, perturb=()):
    """rnn_cluster_kernel: h [B, H] . R [GH, H]^T as one fma chain per output over k = 0 .. Hp - 1 (zeros past H), from
    +0; "desc" runs the chain backwards"""
    B, H = h.shape
    Hp = _r4(H)
    hp = np.zeros((B, Hp), F32)
    hp[:, :H] = h
    Rp = np.zeros((R.shape[0], Hp), F32)
    Rp[:, :H] = R
    acc = np.zeros((B, R.shape[0]), F32)
    for k in (range(Hp - 1, -1, -1) if "desc" in perturb else range(Hp)):
        acc = _fma(hp[:, k, None], Rp[None, :, k], acc)
    return acc


def product_skinny(h, R, perturb=()):
    """skinny_f32_kernel over K = round_up(H, 4) (zero padding): K in chunks of kc = min(K, 1024); lane l of a warp owns
    the float4 groups c = l + 32 it (it < 8) of each chunk and runs one fma chain, x y z w within a group, across its
    groups and the chunks; reduce_scatter_warp then combines the lanes.  Each of its steps adds a lane's value and its
    xor partner's (a commutative f32 add), at xor 16, 8, 4, 2, 1: the same sums as an xor butterfly in that order.
    "butterfly" swaps the first two levels."""
    B, H = h.shape
    K = _r4(H)
    hp = np.zeros((B, K), F32)
    hp[:, :H] = h
    Rp = np.zeros((R.shape[0], K), F32)
    Rp[:, :H] = R
    kc = min(K, 1024)
    lanes = np.arange(32)
    acc = np.zeros((B, R.shape[0], 32), F32)
    for k0 in range(0, K, kc):
        q4 = min(kc, K - k0) // 4
        for it in range(8):
            c = lanes + 32 * it
            live = c < q4
            if not live.any():
                break
            for comp in range(4):
                kk = np.where(live, k0 + 4 * c + comp, 0)
                upd = _fma(hp[:, None, kk], Rp[None, :, kk], acc)
                acc = np.where(live, upd, acc)
    for o in ((8, 16, 4, 2, 1) if "butterfly" in perturb else (16, 8, 4, 2, 1)):
        acc = acc + acc[..., lanes ^ o]
    return acc[..., 0]


def product_f64(h, R):
    return (h.astype(np.float64) @ R.astype(np.float64).T).astype(F32)


def rnn_model(op, x, w, r, b=None, h0=None, c0=None, direction="forward", path="cluster", tanhf=None, perturb=()):
    """(Y, Y_h[, Y_c]) in float32.  path: "cluster" (fma chain), "skinny" or "wgmma" (a float64 product rounded once).
    tanhf(c): the LSTM's last tanh (default: np.tanh in float32, which the CPU test uses).  perturb: "desc" (chain
    backwards), "gru-bias-late" (GRU's input bias of the h gate added after s_h * r), "lstm-rb-early" (the LSTM's
    recurrent bias added before h R), "tanh-ref" (the vecmath tanh for tanhf), "butterfly" (skinny levels swapped)."""
    from oracle import oracle
    from oracle import rnn as orn
    G = 3 if op == "gru" else 4
    x, w, r = (np.asarray(a, F32) for a in (x, w, r))
    T, B, _ = x.shape
    dirs, GH, H = r.shape
    if "tanh-ref" in perturb:
        tanhf = oracle.tanh
    elif tanhf is None:
        tanhf = lambda v: np.tanh(v).astype(F32)  # noqa: E731
    xp = np.einsum("tbi,dgi->tbdg", x.astype(np.float64), w.astype(np.float64))
    xp32 = xp.astype(F32)
    if path != "wgmma":
        assert np.array_equal(xp32, xp), "the input projection is not exact in f32"
    h = np.zeros((dirs, B, H), F32) if h0 is None else np.array(h0, F32)
    c = np.zeros((dirs, B, H), F32) if c0 is None else np.array(c0, F32)
    Y = np.zeros((T, dirs, B, H), F32)
    prod = {"cluster": lambda a, m: product_chain(a, m, perturb), "skinny": lambda a, m: product_skinny(a, m, perturb),
            "wgmma": product_f64}[path]
    sig, tnh = orn.sigmoid, oracle.tanh
    for s in range(T):
        ts = [T - 1 - s if (d == 0 and direction == "reverse") or d == 1 else s for d in range(dirs)]
        cn = []
        for d in range(dirs):
            xg, rec = xp32[ts[d], :, d], prod(h[d], r[d])
            wb = None if b is None else np.asarray(b[d, :GH], F32)
            rb = None if b is None else np.asarray(b[d, GH:], F32)
            if op == "gru":
                gx = xg if wb is None else xg + wb
                sr = rec if rb is None else rec + rb
                z = sig(gx[:, :H] + sr[:, :H])
                rr = sig(gx[:, H:2 * H] + sr[:, H:2 * H])
                if "gru-bias-late" in perturb and wb is not None:
                    ht = tnh((xg[:, 2 * H:] + sr[:, 2 * H:] * rr) + wb[2 * H:])
                else:
                    ht = tnh(gx[:, 2 * H:] + sr[:, 2 * H:] * rr)
                h[d] = (F32(1) - z) * ht + z * h[d]
                Y[ts[d], d] = h[d]
            else:
                v = xg if wb is None else xg + wb
                if "lstm-rb-early" in perturb and rb is not None:
                    v = (v + rb) + rec
                else:
                    v = v + rec
                    v = v if rb is None else v + rb
                i, o, f = sig(v[:, :H]), sig(v[:, H:2 * H]), sig(v[:, 2 * H:3 * H])
                c[d] = f * c[d] + i * tnh(v[:, 3 * H:])
                cn.append(o)
        if op == "lstm":  # one tanhf call per step, on every direction's c
            th = np.asarray(tanhf(c), F32).reshape(c.shape)
            for d in range(dirs):
                h[d] = cn[d] * th[d]
                Y[ts[d], d] = h[d]
    return (Y, h, c) if op == "lstm" else (Y, h)


def model_path(s, rule, ran_cluster):
    if ran_cluster:
        return "cluster"
    return "skinny" if s["B"] <= 32 else "wgmma"


# ---- the LSTM's tanhf, probed ------------------------------------------------------------------------------------------
PROBE_H = 64


def tanhf_probe(rt, ctx, c, per_step=False):
    """tanhf of every element of `c`, as the LSTM kernels compute it: one forward LSTM step with W = R = 0 (I = 0), input
    biases i = -200, o = f = +200, c = 0, h0 = 0 and c0 = the values, on the cluster path or (`per_step`) the per-step
    path.  Then i = 0, f = o = 1 and c~ = 0 exactly, so Y_h = tanhf(c0) bit for bit.  c0 = -0 would come back as +0
    (c = f c0 + i c~ = -0 + 0): zeros are not sent, and tanhf(+-0) = +-0 is returned for them."""
    c = np.asarray(c, F32)
    flat = c.ravel()
    n = flat.size
    if n == 0:
        return c.copy()
    H = PROBE_H
    B = max(1, _cdiv(n, H))
    vals = np.zeros(B * H, F32)
    vals[:n] = np.where(flat == 0, F32(0), flat)
    b = np.zeros((1, 8 * H), F32)
    b[0, :H], b[0, H:3 * H] = -200, 200
    o = rt.LSTM("forward", H)
    ctx.set_f32_mode(True)
    with gc.switches(RTEN_B200_NO_RNN_CLUSTER=1 if per_step else None):
        yh = o.run(ctx, np.zeros((1, B, 0), F32), np.zeros((1, 4 * H, 0), F32), np.zeros((1, 4 * H, H), F32), b=b,
                   initial_c=vals.reshape(1, B, H), outputs=(1,))[1].numpy()
    return np.where(flat == 0, flat, yh.ravel()[:n]).reshape(c.shape)


# ---- fixtures ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def rt():
    import rten_b200
    from rten_b200 import _lib
    _lib.load()
    return rten_b200


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- kernel identity --------------------------------------------------------------------------------------------------
def _kernel_probe():
    import torch
    import rten_b200 as rt
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctx = rt.Context(0)
    res = {}
    for s in specs(n_sms):
        inp = prepare(s)
        args = device_args(ctx, s, inp)

        def call():
            run_case(rt, ctx, s, inp, args)
            ctx.sync()
        for _ in range(3):  # a capture with no kernel record at all is taken again (see rk.capture_kernels)
            got = dk._launches(call, smem=True)
            if got:
                break
        res[spec_id(s)] = got
    print(json.dumps({"sms": n_sms, "launches": res}))


def _family(name):
    for fam in ("umma", "tf32x3", "nd_copy"):
        if f"{fam}_" in name:
            return fam
    return None


def _check_launches(s, r, got):
    """None when `got` is what rule `r` names for the path it took, else a description; (path taken, error)"""
    ours = [((kernel_key(n) or kernel_key(n, STEP_KERNELS)), g, b, sm) for n, g, b, sm in got]
    mine = [(k, g, b, sm) for k, g, b, sm in ours if k is not None]
    counts = {}
    for n, _, _, _ in got:
        f = _family(n)
        if f:
            counts[f] = counts.get(f, 0) + 1
    proj = projection_launches(s)
    if any(b != THREADS for _, _, b, _ in mine if b is not None):
        return None, f"blocks {[b for _, _, b, _ in mine]}"
    if r["path"] == "cluster" and [k for k, _, _, _ in mine] == [("rnn_cluster_kernel", (int(s["op"] == "gru"), r["plan"]["BT"]))]:
        _, g, _, sm = mine[0]
        if g != r["plan"]["grid"]:
            return "cluster", f"grid {g}, rule {r['plan']['grid']}"
        if sm is not None and int(sm) != r["plan"]["smem"]:
            return "cluster", f"shared memory {sm}, rule {r['plan']['smem']}"
        if counts != {k: v for k, v in proj.items() if v}:
            return "cluster", f"other kernels {counts}, projection {proj}"
        return "cluster", None
    if r["path"] == "cluster" and r["plan"]["C"] < 16:
        return None, f"ran {[k for k, _, _, _ in mine]}"
    want = sorted((k, g) for k, g in r["launches"])
    have = sorted((k, g) for k, g, _, _ in mine)
    if have != want:
        return "per-step", f"ran {have[:6]}, rule {want[:6]}"
    others = {k: proj[k] + (r["others"][k] if r["path"] != "init" else 0) for k in proj}
    if counts != {k: v for k, v in others.items() if v}:
        return "per-step", f"other kernels {counts}, rule {others}"
    return ("init" if r["path"] == "init" else "per-step"), None


def test_kernel_identity():
    out = rk.probe_in_child("test_gpu_rnn_kernels")
    n_sms, launches = out["sms"], out["launches"]
    seen, wrong, fell_back, ran16, no_smem = {}, [], [], [], 0
    for s in specs(n_sms):
        sid = spec_id(s)
        r = case_rule(s, n_sms)
        took, err = _check_launches(s, r, launches[sid])
        if err:
            wrong.append((sid, err))
            continue
        if r["plan"] and r["plan"]["C"] == 16:
            (ran16 if took == "cluster" else fell_back).append(sid)
        if took == "cluster":
            no_smem += all(x[3] is None for x in launches[sid])
            k = ("rnn_cluster_kernel", (int(s["op"] == "gru"), r["plan"]["BT"]))
            seen[k] = seen.get(k, 0) + 1
        else:
            for k in {k for k, _ in r["launches"] if k[0] in KERNELS}:
                seen[k] = seen.get(k, 0) + 1
    assert not wrong, f"{len(wrong)} cases ran other kernels or grids than the rule names: {wrong[:6]}"
    missing = [(k, a) for k, args in VARIANTS.items() for a in args if seen.get((k, a), 0) < 2]
    assert not missing, f"instances that fewer than two cases ran: {missing}"
    assert not coverage_gaps(n_sms)
    total = sum(len(v) for v in VARIANTS.values())
    print(f"{total} of {total} instances ran, each at least twice, on {n_sms} SMs; 16-CTA clusters: "
          f"{len(ran16)} scheduled, {len(fell_back)} fell back to the per-step path"
          + (" (Kineto recorded no shared memory)" if no_smem else ""))


# ---- values -----------------------------------------------------------------------------------------------------------
def _ran_cluster(rt, ctx, s, inp, args, r):
    """whether the call ran the cluster kernel: a 16-CTA plan may not schedule, and then the call launches as many
    kernels as the forced per-step path does (the cluster path launches the projection's and one)"""
    if r["path"] != "cluster":
        return False
    if r["plan"]["C"] < 16:
        return True
    n0 = ctx.launches
    run_case(rt, ctx, s, inp, args)
    n1 = ctx.launches
    run_case(rt, ctx, dict(s, step=True), inp, args)
    return n1 - n0 < ctx.launches - n1


def expected(rt, ctx, s, inp, path, perturb=()):
    per_step = path != "cluster"
    tf = (lambda c: tanhf_probe(rt, ctx, c, per_step)) if s["op"] == "lstm" else None  # noqa: E731
    return rnn_model(s["op"], inp["x"], inp["w"], inp["r"], inp["b"], inp["h0"], inp["c0"], s["dir"], path, tf, perturb)


def _check(got, want, s, what, exact=True):
    dirs, T = _dirs(s), s["T"]
    names = ("Y", "Y_h", "Y_c")
    for g, w, nm in zip(got, want, names):
        assert np.isfinite(g).all(), f"{what}: {nm} holds NaN or inf (read outside a view?)"
        if exact:
            gc.assert_bit_exact(g, w, f"{what}: {nm}")
        else:
            d = float(np.abs(g.astype(np.float64) - w).max()) if g.size else 0.0
            assert d <= WGMMA_BOUND, f"{what}: {nm} max |d| {d:.3e} > {WGMMA_BOUND}"
    if T:
        Y, yh = got[0], got[1]
        for d in range(dirs):
            last = 0 if (d == 1 or s["dir"] == "reverse") else T - 1
            gc.assert_bit_exact(yh[d], Y[last, d], f"{what}: Y_h direction {d} against Y at its last step")


def test_values_bit_exact(rt, sms):
    ctx = rt.Context(0)
    worst = 0.0
    for s in specs(sms):
        r = case_rule(s, sms)
        inp = prepare(s)
        args = device_args(ctx, s, inp)
        ran = _ran_cluster(rt, ctx, s, inp, args, r)
        path = model_path(s, r, ran)
        got = run_case(rt, ctx, s, inp, args)
        want = expected(rt, ctx, s, inp, path)
        _check(got, want, s, f"{spec_id(s)} ({path})", exact=path != "wgmma")
        if path == "wgmma":
            worst = max(worst, max(float(np.abs(g.astype(np.float64) - w).max()) for g, w in zip(got, want) if g.size))
    print(f"per-step wgmma product: max |GPU - model| {worst:.2e} (bound {WGMMA_BOUND})")


def test_wgmma_path_reruns_and_replays(rt, sms):
    """The 3xTF32 product is not exact, but it is deterministic: a rerun and a replayed CUDA graph give the same bits"""
    ctx = rt.Context(0)
    cases = [s for s in specs(sms) if case_rule(s, sms)["path"] == "per-step" and s["B"] > 32][:2]
    assert len(cases) == 2
    for s in cases:
        inp = prepare(s)
        d = {k: ctx.to_device(v) for k, v in inp.items() if v is not None}
        args = dict(r=d["r"], b=d.get("b"), initial_h=d.get("h0"))
        if s["op"] == "lstm":
            args["initial_c"] = d.get("c0")
        args = {k: v for k, v in args.items() if v is not None}
        ctx.set_f32_mode(s.get("x3", True))
        o = rt.GRU(s["dir"], s["H"]) if s["op"] == "gru" else rt.LSTM(s["dir"], s["H"])
        kw = {k: v for k, v in args.items() if k != "r"}
        def call():
            with gc.switches(RTEN_B200_NO_RNN_CLUSTER=1 if s.get("step") else None):
                return o.run(ctx, d["x"], d["w"], d["r"], **kw)
        first = [t.numpy() for t in call()]
        again = [t.numpy() for t in call()]
        for a, b in zip(again, first):
            gc.assert_bit_exact(a, b, f"{spec_id(s)}: rerun")
        ctx.sync()
        ctx.graph_begin()
        cap = call()
        graph = ctx.graph_end()
        for i in range(2):
            graph.launch()
            ctx.sync()
            for a, b in zip(cap, first):
                gc.assert_bit_exact(a.numpy(), b, f"{spec_id(s)}: graph replay {i + 1}")


def test_the_comparison_has_teeth(rt, sms):
    """Each deliberate slip in the model changes its bits on a case where the GPU matches the unperturbed model, so the
    bit-exact comparisons above would see the same slip in a kernel"""
    ctx = rt.Context(0)
    all_specs = specs(sms)
    pick = {"gru cluster": next(s for s in all_specs if s["op"] == "gru" and s.get("bias", True) and s["T"] > 1
                                and case_rule(s, sms)["path"] == "cluster" and case_rule(s, sms)["plan"]["C"] == 2),
            "lstm cluster": next(s for s in all_specs if s["op"] == "lstm" and s.get("bias", True) and s["T"] > 1
                                 and case_rule(s, sms)["path"] == "cluster" and case_rule(s, sms)["plan"]["C"] == 2),
            # K >= 128: every lane of the skinny reduction holds part of the sum, so its levels do not commute
            "skinny": next(s for s in all_specs if case_rule(s, sms)["path"] == "per-step" and s["B"] <= 32 and s["H"] >= 128)}
    slips = {"gru cluster": ("desc", "gru-bias-late"), "lstm cluster": ("desc", "lstm-rb-early", "tanh-ref"),
             "skinny": ("butterfly",)}
    for label, s in pick.items():
        inp = prepare(s)
        path = "cluster" if label != "skinny" else "skinny"
        got = run_case(rt, ctx, s, inp)
        want = expected(rt, ctx, s, inp, path)
        for g, w in zip(got, want):
            gc.assert_bit_exact(g, w, f"{label}: {spec_id(s)}")
        for p in slips[label]:
            slipped = expected(rt, ctx, s, inp, path, perturb=(p,))
            assert not all(np.array_equal(g.view(np.int32), w.view(np.int32)) for g, w in zip(got, slipped)), (
                f"{label}: the slip {p!r} leaves the model's bits unchanged")


# ---- the probe itself -------------------------------------------------------------------------------------------------
def test_tanhf_probe_against_float64(rt):
    """The LSTM's tanhf over 10^7 float32 values in [-10, 10] (evenly spaced bit patterns and uniform draws), subnormals,
    +-inf and NaN, against tanh in extended precision: within CUDA's documented 2 ulp; the number of values not
    correctly rounded is printed.  The per-step gate kernel's tanhf gives the same bits on a subset."""
    ctx = rt.Context(0)
    r = _rng("tanhf sweep")
    ten = int(F32(10).view(np.uint32))  # the bit patterns of (0, 10], and of [-10, 0) with the sign bit set
    pos = np.linspace(1, ten, 3_000_000).astype(np.uint32).view(F32)
    neg = -pos
    uni = r.uniform(-10, 10, 4_000_000).astype(F32)
    sub = np.concatenate([np.arange(1, 5001, dtype=np.uint32), np.uint32(0x007FFFFF) - np.arange(5000, dtype=np.uint32)]).view(F32)
    special = np.array([np.inf, -np.inf, np.nan, np.finfo(F32).tiny, -np.finfo(F32).tiny, 9.0, -9.0, 1e-3, 20.0, -20.0], F32)
    x = np.concatenate([neg, pos, uni, sub, -sub, special])
    x = x[~((x == 0) & np.signbit(x))]
    assert x.size >= 10_000_000
    got = tanhf_probe(rt, ctx, x)
    ref = np.tanh(x.astype(np.longdouble))
    nan = np.isnan(x)
    assert np.isnan(got[nan]).all(), "tanhf(NaN) is not NaN"
    assert (got[np.isposinf(x)] == 1).all() and (got[np.isneginf(x)] == -1).all(), "tanhf(+-inf) is not +-1"
    fin = ~nan
    rounded = ref[fin].astype(F32)
    ulp = np.spacing(np.abs(rounded)).astype(np.longdouble)
    err = np.abs(got[fin].astype(np.longdouble) - ref[fin]) / ulp
    bad = int((got[fin].view(np.int32) != rounded.view(np.int32)).sum())
    assert float(err.max()) <= 2.0, f"tanhf error {float(err.max()):.3f} ulp at x = {x[fin][np.argmax(err)]!r}"
    sub_ok = bool((got[np.abs(x) < np.finfo(F32).tiny] == x[np.abs(x) < np.finfo(F32).tiny]).all())
    print(f"tanhf: {x.size} values, max error {float(err.max()):.3f} ulp, {bad} not correctly rounded "
          f"({bad / fin.sum():.2e}); subnormals returned unchanged: {sub_ok}")
    # the gate kernel of the per-step path runs the same tanhf
    part = x[:: max(1, x.size // 200_000)]
    gc.assert_bit_exact(tanhf_probe(rt, ctx, part, per_step=True), got[:: max(1, x.size // 200_000)], "per-step tanhf")
