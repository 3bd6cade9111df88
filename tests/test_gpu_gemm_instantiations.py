"""Every instantiation of the GEMM engine (csrc/gemm_tc.cu, csrc/gemm_simt.cu) against float64, with the kernels each
call must launch.

Which kernel runs is decided on the host at run time: by the engine, the operand layouts, whether fp16 twins are
registered for the weight and bounds for the activation, K % 64, ld % 4 and 16-byte alignment, N >= 8 and K >= 8, and
split-K.  A shape the wgmma engine rejects falls back to the SIMT kernels without a word, and the numbers alone would not
show it.  So every case below names an entry point (linear_act_forward, linear_residual_forward,
linear_act_heads_forward, linear_backward for dW, dX or both with the bias gradient of the layer below), an engine, the
operand form (fp16 twins and both bounds registered, only the bound of x, or nothing), the shape, the strides and the
activation, and the exact set of GEMM-engine kernels the call must launch; the case asserts that set, which
torch.profiler recorded for every case's call in a child process (launched_sets).  Shapes sit on the edges of the 128 x 128 tile (M in {1, 127, 128, 129, 4133}, N in {8, 72, 128, 130,
256, 512}), the k tails of the tf32 form (8, 40, 200) and the fp16 form's 64-k stages (64, 192), with row strides wider
than the rows; each activation runs the bias + activation epilogue (mode 1) and the activation-derivative epilogue of
dX (mode 2) on whole tiles (the straight-line store_tile_whole_act) and on ragged ones (store_tile).  The aux operand of
mode 2 holds the edges of act': ReLU outputs of exactly +0 and -0 and of 1e-30, tanh outputs of exactly +-1 and ELU
outputs one and two float32 ulps above -1.  dW runs with split-K (a short last slice) and without.

Error rule.  Per element, against float64 evaluated on the same float32 inputs,

    |got - ref| <= c * S * max(1, |act'|) + u * |ref|,     S = sum_k |a_k b_k| + |bias| + |aux|

with |bias| where the epilogue adds a bias and |aux| where it adds a residual (mode 3); in mode 2 act' is computed in
float64 from the same float32 aux (it is at most 1 for every activation here).
  c = 4e-6 for the fp32-grade forms (SIMT, the 3-pass tf32 split, the fp16 split).  The 3-pass split keeps ~21
    significant bits of each operand (hi and lo, each 11) and drops lo * lo' (2^-22 of the product); the fp16 split keeps
    22 (hi + lo * 2^-11, both rounded to nearest); so a product errs by at most ~2^-20 of |a b|, 0.24 of c.  The rest of
    c is for fp32 accumulation, which on random operands errs by about 2^-24 of S whatever K is (each partial sum is
    rounded once and the signs are random).  c is 67 * 2^-24: it is not a worst-case bound for adversarial data, whose
    sequential fp32 sum can err by K * 2^-24 of S.
  c = 2^-9 for the single-pass tf32 engine: tf32 truncates each operand to 10 explicit mantissa bits (relative error
    below 2^-10 each), so a product errs by less than 2^-9 of |a b| (first order), and the sum by less than 2^-9 of S.
  u = 2^-21: the epilogue's own roundings -- the bias add, the activation (tanhf is within 2 ulp, the fast ELU of the
    wgmma epilogue within 2.4e-7 absolute), the product with act'.
The head partials of linear_act_heads_forward sum 64 products y_n w_n per row and half tile; against the partials of
float64 y they must hold  sum_n bound(y_n) |w_n| + 1e-5 * sum_n |y_n w_n|  (tests/test_gpu_heads_f16.py's rule for the
sum itself).  The bias gradient db of the layer below is a column sum of the kernel's own dX: within 4e-6 of the sum of
|dX|.
For the 3-pass and fp16 forms the largest error of each output is also at most 4x the SIMT engine's on the same inputs
plus 2^-21 of the largest S: at small k the SIMT engine's fp32 sum is nearly exact, while the split of each operand
leaves up to 2^-21 of it unrepresented (the 3-pass lo half is truncated), an error no accumulation order removes.
Measured on an H100 (80 GB HBM3, 700 W), the 3-pass form's largest error was 10.5x the SIMT engine's at k = 8 and at
most 3.1x from k = 40 up, the fp16 form's at most 1.8x, and the single-pass tf32 engine's error at most 0.56 of its
bound.  A case that must fall back to SIMT under the 3xtf32 engine must give the SIMT engine's bits.
Every case prints its largest error over its bound, and its error over the SIMT engine's where there is one.

test_every_gemm_instantiation_has_a_case (CPU) reads the ptxas reports of an sm_90a build and fails when a compiled
GEMM-engine kernel has no case here and is not on ALLOWLIST, or when a case names a kernel the build lacks."""
import json
import math
import os
import re
import subprocess
import sys

import pytest
import torch

from tests.device_harness import ANY_KERNEL, DEV, Registered, launched, ops_for

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "sample_factory_b200", "csrc", "build")

C_FP32, C_TF32, U = 4e-6, 2.0 ** -9, 2.0 ** -21
C_HEADS = 1e-5
VS_SIMT, VS_SIMT_SPLIT = 4.0, 2.0 ** -21


# ----------------------------------------------------------------------------------------------- the table
def wg(a_mn, b_mn, split3, heads=0, f16=0, res=0):
    """gemm_wgmma_kernel<A_MN, B_MN, SPLIT3, HEADS, F16, RES>"""
    flags = (a_mn, b_mn, split3, heads, f16, res)
    return "gemm_wgmma_kernel<" + ", ".join("true" if f else "false" for f in flags) + ">"


SIMT_FWD = "gemm_simt_kernel<true, true>"     # x K-major, W K-major
SIMT_DW = "gemm_simt_kernel<false, false>"    # dz and x read along their rows
SIMT_DX = "gemm_simt_kernel<true, false>"     # dz K-major, W read along its rows
REDUCE = "splitk_reduce_kernel"
DW16 = "gemm_dw_f16_kernel"
COLSUM = ("colsum_partial_kernel", "colsum_reduce_kernel")
SLAB_M = 65535 * 128 + 1000                   # past the SIMT grid's 65535 row blocks: two row slabs

CASES = []


def case(entry, engine, M, N, K, act, kernels, form=None, **opt):
    """entry: fwd (mode 1), res (mode 3), heads (A = opt["A"] action outputs), dw, dx (mode 2, or 0 for "none"), bwd (dW,
    dX and db of the layer below).  M rows, N outputs, K inputs of the layer (dX is [M, K], dW [N, K]).  form: "f16" (fp16
    twins of W and bounds of x and dz registered), "x_only" (twins, and the bound of x only), None.  opt: ldx, ldc (the
    output's row stride), lddz, ldr, misalign (x starts one float into its buffer)."""
    ks = tuple(name for k in kernels for name in ((k,) if isinstance(k, str) else k))
    strides = "".join(f"-{k}{v}" for k, v in sorted(opt.items()) if k != "A")
    heads = f"-A{opt['A']}" if "A" in opt else ""
    name = f"{entry}-{engine}{'-' + form if form else ''}-{M}x{N}x{K}-{act}{heads}{strides}"
    CASES.append(pytest.param(entry, engine, form, M, N, K, act, ks, opt, id=name))


for s, eng in ((1, "3xtf32"), (0, "tf32")):
    # tf32 form: forward, every activation on whole tiles and on ragged ones; k tails 8, 40, 200
    for M, N, K, act, o in [(1, 8, 8, "elu", {}), (127, 72, 40, "relu", {}), (128, 128, 200, "tanh", {}),
                            (129, 130, 64, "none", {}), (4133, 512, 200, "elu", dict(ldx=264, ldc=520)),
                            (1000, 256, 64, "relu", {}), (256, 128, 40, "none", {}), (300, 256, 8, "tanh", dict(ldc=260))]:
        case("fwd", eng, M, N, K, act, [wg(0, 0, s)], **o)
    # residual: ragged (store_tile_residual) and whole tiles (store_tile_whole<3>)
    case("res", eng, 129, 130, 40, "none", [wg(0, 0, s, res=1)])
    case("res", eng, 256, 256, 64, "none", [wg(0, 0, s, res=1)], ldx=72, ldr=264, ldc=260)
    # head partials
    for M, N, K, act, A in [(1, 128, 8, "elu", 1), (129, 512, 40, "tanh", 8), (1000, 256, 200, "relu", 5),
                            (300, 128, 64, "none", 3)]:
        case("heads", eng, M, N, K, act, [wg(0, 0, s, heads=1)], A=A)
    # dX = dz . W, mode 2 for every activation (mode 0 for none)
    for M, N, K, act, o in [(1, 8, 8, "elu", {}), (127, 40, 72, "relu", {}), (129, 200, 136, "tanh", {}),
                            (1000, 64, 512, "elu", dict(ldx=520, ldc=516, lddz=68)), (300, 40, 256, "relu", {}),
                            (256, 200, 128, "tanh", {}), (300, 64, 128, "none", {})]:
        case("dx", eng, M, N, K, act, [wg(0, 1, s)], **o)
    # dW = dz^T x: one slice (M < 256; 144 tiles), split-K with a short last slice
    case("dw", eng, 100, 72, 40, "none", [wg(1, 1, s)])
    case("dw", eng, 300, 1536, 1536, "none", [wg(1, 1, s)])
    case("dw", eng, 1000, 128, 128, "none", [wg(1, 1, s), REDUCE])
    case("dw", eng, 4133, 130, 200, "none", [wg(1, 1, s), REDUCE], lddz=136, ldx=204)
    case("bwd", eng, 1000, 128, 256, "elu", [wg(1, 1, s), REDUCE, wg(0, 1, s), COLSUM])

# fp16 form: K (the k of the GEMM) a multiple of the 64-k stage, twins and bounds registered
for M, N, K, act, o in [(1, 8, 64, "elu", {}), (129, 130, 192, "relu", {}), (4133, 512, 64, "tanh", dict(ldx=72, ldc=516)),
                        (1000, 256, 192, "none", {}), (300, 128, 64, "elu", {}), (256, 256, 64, "relu", {}),
                        (256, 128, 192, "tanh", {})]:
    case("fwd", "3xtf32", M, N, K, act, [wg(0, 0, 1, f16=1)], "f16", **o)
for M, N, K, act, A in [(1, 128, 64, "elu", 1), (129, 512, 192, "tanh", 8), (1000, 256, 64, "relu", 5),
                        (300, 128, 192, "none", 3)]:
    case("heads", "3xtf32", M, N, K, act, [wg(0, 0, 1, heads=1, f16=1)], "f16", A=A)
for M, N, K, act, o in [(1, 64, 8, "elu", {}), (129, 192, 136, "relu", {}), (1000, 64, 512, "tanh", dict(ldx=520, ldc=516)),
                        (300, 192, 256, "elu", {}), (256, 64, 128, "relu", {}), (256, 192, 256, "tanh", {}),
                        (300, 64, 128, "none", {})]:
    case("dx", "3xtf32", M, N, K, act, [wg(0, 1, 1, f16=1)], "f16", **o)
case("dw", "3xtf32", 100, 72, 40, "none", [DW16], "f16")
case("dw", "3xtf32", 1000, 128, 128, "none", [DW16, REDUCE], "f16")
case("dw", "3xtf32", 4133, 130, 200, "none", [DW16, REDUCE], "f16", lddz=136, ldx=204)
case("bwd", "3xtf32", 1000, 128, 256, "tanh", [DW16, REDUCE, wg(0, 1, 1, f16=1), COLSUM], "f16")

# routing: what the wgmma engine does not take
case("fwd", "3xtf32", 300, 128, 64, "elu", [SIMT_FWD], ldx=66)                 # ld % 4 != 0
case("fwd", "3xtf32", 300, 128, 64, "relu", [SIMT_FWD], misalign=1)            # base not 16-byte aligned
case("fwd", "3xtf32", 300, 64, 4, "tanh", [SIMT_FWD])                          # K < 8
case("fwd", "3xtf32", 300, 4, 64, "elu", [SIMT_FWD])                           # N < 8
case("res", "3xtf32", 300, 128, 64, "none", [SIMT_FWD], ldx=66)
case("bwd", "3xtf32", 300, 64, 40, "elu", [SIMT_DW, REDUCE, SIMT_DX, COLSUM], ldx=42)
case("bwd", "3xtf32", 300, 64, 4, "relu", [SIMT_DW, REDUCE, SIMT_DX, COLSUM])  # dW's N (= K) < 8
case("fwd", "3xtf32", 300, 128, 200, "elu", [wg(0, 0, 1)], "f16")             # K % 64 != 0: the tf32 form
case("heads", "3xtf32", 300, 128, 40, "elu", [wg(0, 0, 1, heads=1)], "f16", A=2)
case("dx", "3xtf32", 300, 40, 128, "relu", [wg(0, 1, 1)], "f16")
case("dx", "3xtf32", 129, 200, 130, "tanh", [SIMT_DX])                        # W's row stride K % 4 != 0
case("res", "3xtf32", 256, 256, 64, "none", [wg(0, 0, 1, res=1)], "f16")       # mode 3 has no fp16 form
case("bwd", "3xtf32", 1000, 128, 256, "elu", [wg(1, 1, 1), REDUCE, wg(0, 1, 1), COLSUM], "x_only")   # dz has no bound

# the SIMT engine
for M, N, K, act, o in [(1, 8, 4, "elu", {}), (129, 130, 37, "relu", dict(ldx=40, ldc=132)), (300, 70, 37, "tanh", {}),
                        (128, 64, 16, "none", {})]:
    case("fwd", "simt", M, N, K, act, [SIMT_FWD], **o)
case("res", "simt", 129, 130, 40, "none", [SIMT_FWD])
case("dx", "simt", 127, 40, 72, "relu", [SIMT_DX])
case("dx", "simt", 300, 64, 128, "tanh", [SIMT_DX], ldx=132)
case("dw", "simt", 100, 72, 40, "none", [SIMT_DW])
case("bwd", "simt", 1000, 128, 256, "elu", [SIMT_DW, REDUCE, SIMT_DX, COLSUM])    # split-K with the dW epilogue
case("fwd", "simt", SLAB_M, 8, 8, "elu", [SIMT_FWD])                               # row slabs
case("res", "simt", SLAB_M, 8, 8, "none", [SIMT_FWD])                              # ... with aux offset per slab

# compiled, reached by no entry point
ALLOWLIST = {
    wg(1, 0, 1): "gemm_tc's (a_mn, !b_mn) branch: no entry point reads an MN-major A against a K-major B",
    wg(1, 0, 0): "gemm_tc's (a_mn, !b_mn) branch: no entry point reads an MN-major A against a K-major B",
    "gemm_simt_kernel<false, true>": "gemm_simt's (!a_kcont, b_kcont) branch: no entry point calls it",
}


# ----------------------------------------------------------------------------------------------- the table is complete
def _compiled_kernels():
    names = []
    for log in ("gemm_tc", "gemm_simt"):
        path = os.path.join(BUILD, f"{log}.ptxas.log")
        assert os.path.isfile(path), f"{path} missing: build the library first (__graft_entry__.build())"
        names += re.findall(r"Function properties for (\S+)", open(path).read())
    demangled = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True,
                               check=True).stdout.splitlines()
    return {m.group(1) for n in demangled for m in [re.match(rf"(?:void )?sfb::({ANY_KERNEL})\(", n)] if m}


def test_every_gemm_instantiation_has_a_case():
    compiled = _compiled_kernels()
    assert any(k.startswith("gemm_wgmma_kernel<") for k in compiled) and SIMT_FWD in compiled, sorted(compiled)
    named = {k for c in CASES for k in c.values[7]}
    covered = named | set(ALLOWLIST)
    assert not compiled - covered, f"GEMM kernels with no case in this table: {sorted(compiled - covered)}"
    assert not covered - compiled, f"cases name kernels the build does not have: {sorted(covered - compiled)}"
    assert not named & set(ALLOWLIST), f"allowlisted kernels with a case: {sorted(named & set(ALLOWLIST))}"


# ----------------------------------------------------------------------------------------------- inputs
def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _view(rows, cols, ld, gen, scale=1.0, misalign=0, edit=None):
    """[rows, cols] view of a [rows, ld] device buffer of normal values (the columns past `cols` hold data too)"""
    buf = torch.randn(rows, max(ld or cols, cols) + misalign, generator=gen, device=DEV) * scale
    if edit is not None:
        edit(buf)
    return buf, buf[:, misalign:misalign + cols]


def _activations(act):
    """edit of a buffer into float32 outputs of `act`, with the edges of act' (its derivative from the output)"""
    def edit(buf):
        flat = buf.view(-1)
        if act == "elu":
            flat.copy_(torch.nn.functional.elu(flat))
            flat[::5] = -1.0 + 2.0 ** -24          # one ulp above -1: act' = 2^-24
            flat[2::7] = -1.0 + 2.0 ** -23
        elif act == "relu":
            flat.clamp_(min=0.0)                   # act' = 0 at exactly 0
            flat[::5] = -0.0
            flat[2::7] = 1e-30                     # act' = 1
        elif act == "tanh":
            flat.copy_(torch.tanh(flat))
            flat[::5] = 1.0                        # act' = 0
            flat[2::7] = -1.0
    return edit


def _inputs(entry, form, M, N, K, act, opt):
    gen = _gen(M + 7 * N + 31 * K + len(act))
    d = {}
    x_edit = _activations(act) if entry in ("dx", "bwd") else None
    d["xbuf"], d["x"] = _view(M, K, opt.get("ldx"), gen, misalign=opt.get("misalign", 0), edit=x_edit)
    d["W"] = (torch.randn(N, K, generator=gen, device=DEV) / math.sqrt(K)).contiguous()
    d["b"] = torch.randn(N, generator=gen, device=DEV) * 0.1
    if entry in ("dw", "dx", "bwd"):
        d["dzbuf"], d["dz"] = _view(M, N, opt.get("lddz"), gen, scale=0.1)
    if entry == "res":
        d["rbuf"], d["r"] = _view(M, N, opt.get("ldr"), gen)
    if entry == "heads":
        A = opt["A"]
        d["Wv"] = torch.randn(N, generator=gen, device=DEV) / math.sqrt(N)
        d["Wa"] = (torch.randn(A, N, generator=gen, device=DEV) / math.sqrt(N)).contiguous()
    return d


def _nan(rows, cols, ld=None):
    return torch.full((rows, ld or cols), float("nan"), device=DEV)[:, :cols]


def _outputs(entry, M, N, K, opt, engine):
    ops = ops_for()
    o = {}
    if entry in ("fwd", "res", "heads"):
        o["y"] = _nan(M, N, opt.get("ldc"))
    if entry == "heads":
        P = ops.linear_heads_partials(N, opt["A"], ops.ENGINES[engine])
        o["part"] = torch.full((P, M, ops.HEAD_PART_PAD), float("nan"), device=DEV)
    if entry in ("dw", "bwd"):
        o["dW"] = torch.full((N, K), float("nan"), device=DEV)
    if entry in ("dx", "bwd"):
        o["dx"] = _nan(M, K, opt.get("ldc"))
    if entry == "bwd":
        o["db"] = torch.full((K,), float("nan"), device=DEV)
    return o


def _call(entry, engine, d, o, act, M, N, K):
    """the entry point's call, on preallocated inputs and outputs (what runs under the profiler)"""
    ops = ops_for()
    e, a = ops.ENGINES[engine], ops.ACT[act]
    if entry == "fwd":
        return lambda: ops.linear_act_forward(d["x"], d["W"], d["b"], o["y"], a, e)
    if entry == "res":
        return lambda: ops.linear_residual_forward(d["x"], d["W"], d["b"], d["r"], o["y"], e)
    if entry == "heads":
        return lambda: ops.linear_act_heads_forward(d["x"], d["W"], d["b"], o["y"], a, e, d["Wv"], d["Wa"], o["part"])
    ws = torch.empty(ops.linear_backward_workspace_bytes(M, N, K) // 4 + 4, device=DEV)
    return lambda: ops.linear_backward(d["dz"], d["x"], d["W"], a, o.get("dW"), o.get("dx"), o.get("db"), e, ws)


def _run(entry, engine, form, d, act, M, N, K, opt, kernels=None):
    """outputs of the entry point under `engine`; with `kernels`, (outputs, the GEMM-engine kernels the call launched,
    profiled in the hope of exactly `kernels`)"""
    o = _outputs(entry, M, N, K, opt, engine)
    fn = _call(entry, engine, d, o, act, M, N, K)
    reg = None
    if form is not None:   # bounds over the whole buffers the (strided) operands lie in
        reg = Registered(d["W"], x=d["xbuf"], dz=d.get("dzbuf") if form == "f16" else None)
    try:
        got = fn() if kernels is None else launched(fn, names=ANY_KERNEL, expected=kernels)
        torch.cuda.synchronize()
    finally:
        if reg is not None:
            reg.__exit__(None, None, None)
    return o if kernels is None else (o, got)


def print_launched_sets():
    """JSON {case id: the kernels its call launched} on stdout, every case's call profiled once in this process"""
    ops = ops_for()
    out = {}
    for p in CASES:
        entry, engine, form, M, N, K, act, kernels, opt = p.values
        if engine != "simt" and not ops.tc_available():
            continue
        d = _inputs(entry, form, M, N, K, act, opt)
        out[p.id] = sorted(_run(entry, engine, form, d, act, M, N, K, opt, kernels)[1])
        del d
        torch.cuda.empty_cache()
    print(json.dumps(out))


@pytest.fixture(scope="module")
def launched_sets():
    """the launched kernels of every case, profiled in a process of its own: profiler sessions leave state behind in the
    process that runs them, and after this table's ~100 sessions, with heavy device work between them, later profiles in
    the same process (other modules' tables) lost their device records"""
    ops_for()
    code = "from tests.test_gpu_gemm_instantiations import print_launched_sets; print_launched_sets()"
    res = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=1200)
    assert res.returncode == 0, res.stderr[-3000:]
    return json.loads(res.stdout.strip().splitlines()[-1])


# ----------------------------------------------------------------------------------------------- float64 references
def _act64(z, act):
    if act == "elu":
        return torch.where(z > 0, z, torch.expm1(z))
    if act == "relu":
        return z.clamp_min(0.0)
    if act == "tanh":
        return torch.tanh(z)
    return z


def _dact64(h, act):
    """act' from the activation's output h (float64 of the float32 aux)"""
    if act == "elu":
        return torch.where(h > 0, torch.ones_like(h), h + 1.0)
    if act == "relu":
        return (h > 0).double()
    if act == "tanh":
        return 1.0 - h * h
    return torch.ones_like(h)


def _references(entry, d, act, c):
    """{output: (ref, bound, largest S)} for the outputs that do not depend on another output of the kernel"""
    f = {k: v.double() for k, v in d.items() if k in ("x", "W", "b", "dz", "r", "Wv", "Wa")}
    a = {k: v.abs() for k, v in f.items()}
    out = {}
    if entry in ("fwd", "heads"):
        ref, S = _act64(f["x"] @ f["W"].t() + f["b"], act), a["x"] @ a["W"].t() + a["b"]
    if entry == "res":
        ref, S = f["x"] @ f["W"].t() + f["b"] + f["r"], a["x"] @ a["W"].t() + a["b"] + a["r"]
    if entry in ("fwd", "heads", "res"):
        out["y"] = (ref, c * S + U * ref.abs(), S.max().item())
    if entry in ("dw", "bwd"):
        ref, S = f["dz"].t() @ f["x"], a["dz"].t() @ a["x"]
        out["dW"] = (ref, c * S + U * ref.abs(), S.max().item())
    if entry in ("dx", "bwd"):
        dact = _dact64(f["x"], act)
        ref, S = (f["dz"] @ f["W"]) * dact, a["dz"] @ a["W"]
        out["dx"] = (ref, c * S * dact.abs().clamp_min(1.0) + U * ref.abs(), S.max().item())
    return out


def _check(what, got, ref, bound):
    """asserts |got - ref| <= bound elementwise; returns (largest |error|, largest |error| / bound)"""
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)                     # (NaN fails)
    idx = bad.nonzero()[:5].tolist()
    assert not bad.any(), (f"{what}: {int(bad.sum())} elements beyond the bound, e.g. at {idx}: got "
                           f"{[got[tuple(i)].item() for i in idx]}, ref {[ref[tuple(i)].item() for i in idx]}, bound "
                           f"{[bound[tuple(i)].item() for i in idx]}")
    ratio = (err / bound.clamp_min(1e-300)).max().item()
    return err.max().item(), ratio


# ----------------------------------------------------------------------------------------------- the cases
def _fallback(kernels):
    return not any(k.startswith("gemm_wgmma_kernel") or k == DW16 for k in kernels)


@pytest.mark.gpu
@pytest.mark.parametrize("entry,engine,form,M,N,K,act,kernels,opt", CASES)
def test_gemm_instantiation(entry, engine, form, M, N, K, act, kernels, opt, launched_sets, request):
    ops_for(engine)
    d = _inputs(entry, form, M, N, K, act, opt)
    ran = launched_sets[request.node.callspec.id]
    assert set(ran) == set(kernels), f"launched {ran}, expected {sorted(kernels)}"
    got = _run(entry, engine, form, d, act, M, N, K, opt)
    c = C_TF32 if engine == "tf32" else C_FP32
    refs = _references(entry, d, act, c)
    errs, report = {}, []
    for k, (ref, bound, _) in refs.items():
        errs[k], ratio = _check(f"{k}", got[k], ref, bound)
        report.append(f"{k} err/bound {ratio:.3g}")
    if entry == "heads":
        A, P = opt["A"], got["part"].shape[0]
        ref_y, bound_y, _ = refs["y"]
        Wh = torch.cat([d["Wv"].view(1, N), d["Wa"]]).double()
        part = lambda y, w: torch.einsum("mpk,apk->pma", y.reshape(M, P, 64), w.reshape(A + 1, P, 64))  # noqa: E731
        ref_p = part(ref_y, Wh)
        bound_p = part(bound_y, Wh.abs()) + C_HEADS * part(ref_y.abs(), Wh.abs())
        _, ratio = _check("head partials", got["part"][:, :, :A + 1], ref_p, bound_p)
        report.append(f"partials err/bound {ratio:.3g}")
        assert torch.all(got["part"][:, :, A + 1:] == 0), "padding columns of the partials"
    if entry == "bwd":
        dx = got["dx"].double()
        _, ratio = _check("db", got["db"], dx.sum(0), C_FP32 * dx.abs().sum(0) + U * dx.sum(0).abs())
        report.append(f"db err/bound {ratio:.3g}")
    if engine == "3xtf32":
        simt_entry = "fwd" if entry == "heads" else entry
        simt = _run(simt_entry, "simt", None, d, act, M, N, K, opt)
        for k in errs:
            if _fallback(kernels):
                assert torch.equal(got[k], simt[k]), f"{k}: the fallback must give the SIMT engine's bits"
                continue
            ref = refs[k][0]
            e_simt = (simt[k].double() - ref).abs().max().item()
            limit = VS_SIMT * e_simt + VS_SIMT_SPLIT * refs[k][2]
            assert errs[k] <= limit, f"{k}: largest error {errs[k]:.3g}, SIMT engine's {e_simt:.3g}"
            report.append(f"{k} err/simt {errs[k] / max(e_simt, 1e-300):.3g}")
    print(f"[gemm] {entry}-{engine}-{form}-{M}x{N}x{K}-{act}: " + ", ".join(report))
