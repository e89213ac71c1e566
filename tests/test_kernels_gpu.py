"""Kernel-level tests: the projection (GEMV, tiled wgmma, stream-K wgmma), paged-attention, norm and argmax kernels run one
at a time through tests/kernel_shim.cpp and are compared with a float64 reference computed on the CPU.

Exact inputs.  Weights, activations, q and k are small dyadic values (integers in [-8, 8] times 2^-4; q times 2^-3).  Every
product is then a multiple of 2^-8 (2^-7 for q.k), every partial sum stays below 2^13 even at K = 28672, and so every fp32
summation order (GEMV FMAs, wgmma k-blocks, the stream-K fix-up) gives exactly the float64 result:
  - EPI_F32 must equal the float64 product bit for bit;
  - every bf16 epilogue must equal a float32 emulation of its rounding points (csrc/epilogue.cuh) applied to that exact
    accumulator, bit for bit; SWIGLU calls expf and may differ from the host's libm by 1 bf16 ulp on a few elements, and
    GELU is bounded against float64 (`assert_gelu`);
  - attention scores bf16(bf16(q.k) * scale) are exact, so only the fp32 softmax, __expf and the final rounding remain
    (bounds at `attn_bound`).
Toleranced comparisons are each paired with a negative control: the same check must reject a deliberately wrong reference
(a dropped key, a split counted twice, a dropped k-block, a RoPE position shifted by one).

The stream-K owner CTA spin-waits on higher-numbered CTAs, so no launch here asks for more CTAs than the device has SMs.
"""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "substratus_b200", "csrc")
LIBDIR = os.path.join(ROOT, "substratus_b200", "lib")
DEV = "cuda:0"

EPI_F32, EPI_F32_BF16R, EPI_RESID, EPI_SWIGLU, EPI_QKV_ROPE, EPI_BF16, EPI_F32_PUSH, EPI_GELU, EPI_RESID2 = range(9)
NORM_NONE, NORM_RMS, NORM_LN = 0, 1, 2
SENTINEL = 0x5A5A  # bf16 bit pattern the KV caches are filled with before a QKV epilogue writes into them


class ShimProj(C.Structure):
    _fields_ = ([(n, C.c_void_p) for n in ("W", "x", "row_map", "norm_w", "norm_b", "f32_add", "resid", "resid2", "rope_cs",
                                           "block_table", "row_slot", "row_pos", "out_f32", "out_bf16", "q_out", "kcache",
                                           "vcache")]
                + [(n, C.c_int) for n in ("N", "K", "ldx", "M", "ld_out", "q_rows", "kv_rows", "head_dim", "bt_stride",
                                          "block_size", "kvh")]
                + [("eps", C.c_float)])


class ShimAttn(C.Structure):
    _fields_ = ([(n, C.c_void_p) for n in ("q", "kcache", "vcache", "block_table", "row_slot", "row_pos", "tile_row0",
                                           "tile_nrows", "out", "part_o", "part_ml", "counters")]
                + [(n, C.c_int) for n in ("bt_stride", "M", "n_heads", "kvh", "group", "head_dim", "block_size", "n_splits",
                                          "n_tiles")]
                + [("scale", C.c_float)])


def _ptr(t):
    return None if t is None else t.data_ptr()


def _struct(cls, **kw):
    s = cls()
    for k, v in kw.items():
        setattr(s, k, _ptr(v) if isinstance(v, torch.Tensor) else v)
    return s


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    from substratus_b200 import load_library

    load_library()  # the shim's dependency resolves to this already-loaded copy (one static CUDA runtime)
    so = str(tmp_path_factory.mktemp("kernel_shim") / "libkernel_shim.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-shared", "-fPIC", "-I", CSRC, "-I", "/usr/local/cuda/include", "-o", so,
                    os.path.join(ROOT, "tests", "kernel_shim.cpp"), "-L", LIBDIR, "-lsubstratus_b200", "-Wl,-rpath," + LIBDIR],
                   check=True)
    lib = C.CDLL(so)
    vp, i, f = C.c_void_p, C.c_int, C.c_float
    lib.shim_gemv.argtypes = [C.POINTER(ShimProj), i, i, i]
    lib.shim_gemv_pick_bt.argtypes = [i, i]
    lib.shim_tc_gemm.argtypes = [C.POINTER(ShimProj), i, i, i, vp, vp, i]
    lib.shim_attn_decode.argtypes = [C.POINTER(ShimAttn)]
    lib.shim_attn_prefill.argtypes = [C.POINTER(ShimAttn)]
    lib.shim_rmsnorm.argtypes = [vp, vp, vp, i, i, f]
    lib.shim_layernorm.argtypes = [vp, vp, vp, vp, i, i, f]
    lib.shim_argmax.argtypes = [vp, i, i, vp, vp, vp, vp]
    torch.cuda.init()
    return lib


@pytest.fixture(scope="module")
def n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def sk_ws(n_sm):
    """Stream-K workspace as the engine sizes it: 2 slots per SM of 64 x 128 fp32, zeroed flags."""
    slots = 2 * n_sm
    return torch.zeros(slots * 64 * 128, dtype=torch.float32, device=DEV), torch.zeros(slots, dtype=torch.int32, device=DEV), slots


def launch(fn, *args):
    """Run one launcher; synchronise so a fault is reported at the launch that caused it."""
    torch.cuda.synchronize()
    rc = fn(*args)
    torch.cuda.synchronize()
    assert rc == 0, f"{fn.__name__} returned {rc}"


# ------------------------------------------------------------------------------------------------------------ host math
def bf(t):
    """float32 -> nearest bf16 (ties to even) -> float32, on the CPU."""
    return t.float().to(torch.bfloat16).float()


def ulp_bf16(x):
    """Spacing of bf16 numbers at |x| (2^(e-7) for |x| in [2^e, 2^(e+1)))."""
    _, e = torch.frexp(x.abs().double().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(x, dtype=torch.float64), (e - 8).to(torch.int32))


def dyadic(shape, gen, scale=2.0 ** -4):
    return (torch.randint(-8, 9, shape, generator=gen, device=DEV, dtype=torch.int32).float() * scale).to(torch.bfloat16)


def continuous(shape, gen, amp=1.0):
    return (torch.randn(shape, generator=gen, device=DEV) * amp).to(torch.bfloat16)


def matmul64(x, W, rows=None):
    """float64 x[M, K] @ W[N, K]^T on the CPU (x may be gathered by `rows`), in column chunks to bound host memory."""
    xd = x.cpu().double()
    if rows is not None:
        xd = xd[rows.cpu().long()]
    out = torch.empty(xd.shape[0], W.shape[0], dtype=torch.float64)
    for n0 in range(0, W.shape[0], 4096):
        out[:, n0:n0 + 4096] = xd @ W[n0:n0 + 4096].cpu().double().T
    return out


def abs_matmul64(x, W):
    xd = x.cpu().double().abs()
    out = torch.empty(xd.shape[0], W.shape[0], dtype=torch.float64)
    for n0 in range(0, W.shape[0], 4096):
        out[:, n0:n0 + 4096] = xd @ W[n0:n0 + 4096].cpu().double().abs().T
    return out


def epilogue_ref(epi, acc, resid=None, resid2=None, f32_add=None):
    """float32 emulation of gemv_epilogue's rounding points on an fp32 accumulator acc[M, N] (CPU).  Returns float32 for
    the fp32 epilogues, bf16 otherwise."""
    acc = acc.float()
    if epi == EPI_F32:
        return acc + f32_add.cpu().float() if f32_add is not None else acc
    if epi == EPI_F32_BF16R:
        return bf(acc)
    if epi == EPI_BF16:
        return acc.to(torch.bfloat16)
    if epi == EPI_RESID:
        return (bf(acc) + resid.cpu().float()).to(torch.bfloat16)
    if epi == EPI_RESID2:
        return (bf(bf(acc) + resid2.cpu().float()) + resid.cpu().float()).to(torch.bfloat16)
    if epi == EPI_SWIGLU:
        g, u = bf(acc[:, 0::2]), bf(acc[:, 1::2])
        return (bf(g / (1.0 + torch.exp(-g))) * u).to(torch.bfloat16)
    if epi == EPI_GELU:
        g = bf(acc)
        return ((0.5 * g) * (1.0 + torch.erf(g * np.float32(0.70710678118654752440)))).to(torch.bfloat16)
    raise ValueError(epi)


def rope_table(max_pos, D, theta=10000.0):
    """Packed (cos bf16 | sin bf16 << 16) per (position, j), built like Engine::alloc_runtime.  Returns (device int32
    table, cos float32 [max_pos, D/2], sin float32 [max_pos, D/2])."""
    half = D // 2
    inv = 1.0 / np.power(np.float32(theta), np.arange(half, dtype=np.float32) * 2 / np.float32(D), dtype=np.float32)
    ang = (np.arange(max_pos, dtype=np.float32)[:, None] * inv[None, :]).astype(np.float32)
    c = torch.from_numpy(np.cos(ang)).to(torch.bfloat16)
    s = torch.from_numpy(np.sin(ang)).to(torch.bfloat16)
    bits = lambda t: t.view(torch.int16).numpy().astype(np.uint16).astype(np.uint32)
    packed = (bits(c) | (bits(s) << 16)).view(np.int32)
    return torch.from_numpy(packed.copy()).to(DEV), c.float(), s.float()


def rope_ref(x0, x1, c, s):
    """(q*cos) + (rotate_half(q)*sin) on a RoPE pair (j, j + D/2), every op rounded to bf16 (epilogue.cuh)."""
    x0, x1 = bf(x0), bf(x1)
    return bf(bf(x0 * c) + bf(-x1 * s)), bf(bf(x1 * c) + bf(x0 * s))


class KvLayout:
    """Paged KV cache of `slots` sequences: every (slot, logical block) maps to its own physical block, shuffled."""

    def __init__(self, slots, max_pos, bs, kvh, D, gen):
        self.bs, self.kvh, self.D, self.stride = bs, kvh, D, max_pos // bs
        self.n_blocks = slots * self.stride
        perm = torch.randperm(self.n_blocks, generator=gen)
        self.bt = perm.view(slots, self.stride).int()
        self.bt_dev = self.bt.to(DEV)

    def empty_cache(self):
        c = torch.empty(self.n_blocks, self.kvh, self.bs, self.D, dtype=torch.bfloat16, device=DEV)
        c.view(torch.int16).fill_(SENTINEL)
        return c

    def cells(self, slot, pos):
        """physical block and in-block offset of each (slot, pos) (CPU long tensors)"""
        slot, pos = torch.as_tensor(slot).long(), torch.as_tensor(pos).long()
        return self.bt[slot, pos // self.bs].long(), pos % self.bs


def qkv_ref(acc, pos, slot, H, KVH, D, cos, sin, kv: KvLayout, caches=True):
    """QKV_ROPE on acc[M, (H + 2 KVH) D] (pair-interleaved rows): q [M, H D] bf16 and the expected caches (CPU)."""
    M, half = acc.shape[0], D // 2
    acc = acc.float()
    v0, v1 = acc[:, 0::2], acc[:, 1::2]
    c, s = cos[pos.long()][:, None, :], sin[pos.long()][:, None, :]
    qa, qb = rope_ref(v0[:, :H * half].reshape(M, H, half), v1[:, :H * half].reshape(M, H, half), c, s)
    ka, kb = rope_ref(v0[:, H * half:(H + KVH) * half].reshape(M, KVH, half),
                      v1[:, H * half:(H + KVH) * half].reshape(M, KVH, half), c, s)
    q = torch.cat([qa, qb], -1).reshape(M, H * D).to(torch.bfloat16)
    k = torch.cat([ka, kb], -1).to(torch.bfloat16)
    if not caches:
        return q, None, None
    v = acc[:, (H + KVH) * D:].reshape(M, KVH, D).to(torch.bfloat16)
    kc = torch.empty(kv.n_blocks, KVH, kv.bs, D, dtype=torch.bfloat16)
    kc.view(torch.int16).fill_(SENTINEL)
    vc = kc.clone()
    blk, off = kv.cells(slot, pos)
    kc[blk, :, off] = k
    vc[blk, :, off] = v
    return q, kc, vc


def same_bits(a, b):
    a, b = a.cpu(), b.cpu()
    if a.dtype == torch.bfloat16:
        a, b = a.view(torch.int16), b.view(torch.int16)
    elif a.dtype == torch.float32:
        a, b = a.view(torch.int32), b.view(torch.int32)
    return bool(torch.equal(a, b))


def assert_same_bits(got, want, what):
    if same_bits(got, want):
        return
    g, w = got.cpu().double(), want.cpu().double()
    bad = (g != w).nonzero()
    i = tuple(bad[0].tolist())
    raise AssertionError(f"{what}: {bad.shape[0]} of {g.numel()} elements differ; first at {i}: got {g[i].item()!r}, "
                         f"want {w[i].item()!r}; max |diff| {float((g - w).abs().max()):.3e}")


def assert_within_ulp(got, want, what, max_frac):
    """bf16 results that may differ by one ulp (libm expf / erff vs the device's) on at most max_frac of the elements."""
    g, w = got.cpu().float(), want.cpu().float()
    diff = (g - w).abs().double()
    n_bad = int((diff != 0).sum())
    assert bool((diff <= ulp_bf16(w)).all()), f"{what}: max |diff| {float(diff.max()):.3e} exceeds one bf16 ulp"
    assert n_bad <= max_frac * g.numel(), f"{what}: {n_bad} of {g.numel()} elements off by one ulp"


def assert_gelu(got, acc, what):
    """EPI_GELU against float64: y = 0.5 g (1 + erf(g / sqrt 2)) with g = bf16(acc).  erff is within 2 fp32 ulps; near
    erf = -1 an ulp is 2^-24, so in the negative tail the fp32 result carries an absolute error up to |g| 2^-24 that is
    many bf16 ulps of a tiny y.  Bound: ulp_bf16(y) (final rounding) + |g| 2^-22."""
    g = bf(acc.cpu().float()).double()
    y = 0.5 * g * (1.0 + torch.erf(g / math.sqrt(2.0)))
    err = (got.cpu().double() - y).abs() / (ulp_bf16(y) + g.abs() * 2.0 ** -22)
    i = tuple(int(v) for v in torch.nonzero(err == err.max())[0])
    print(f"{what}: GELU max |err| / bound = {float(err.max()):.3f}")
    assert float(err.max()) <= 1.0, f"{what}: at {i} g={g[i].item()!r} got {got.cpu()[i].item()!r} want {y[i].item()!r}"


def proj_bound(x, W):
    """Continuous inputs: |kernel - float64| <= 2^-16 * sum_k |w x| per output (fp32 accumulation in blocks, not one
    running sum of K terms: the error stays within a few hundred fp32 ulps of the absolute sum)."""
    return 2.0 ** -16 * abs_matmul64(x, W)


def within(got, ref, bound):
    return bool(((got.cpu().double() - ref).abs() <= bound).all())


# ------------------------------------------------------------------------------------------------------------ drivers
def run_gemv(shim, epi, norm, n_sm, **kw):
    launch(shim.shim_gemv, C.byref(_struct(ShimProj, **kw)), epi, norm, n_sm)


def run_tc(shim, epi, tn, n_sm, sk=None, **kw):
    part, flags, slots = sk if sk is not None else (None, None, 0)
    launch(shim.shim_tc_gemm, C.byref(_struct(ShimProj, **kw)), epi, tn, n_sm, _ptr(part), _ptr(flags), slots)


def tc_pick_tn(M):
    return 16 if M <= 16 else 32 if M <= 32 else 64 if M <= 64 else 128


def nsm_of(kind, n_sm):
    return n_sm if kind == "all" else min(kind, n_sm)


def run_proj(shim, kernel, epi, n_sm, sk_ws, M, **kw):
    """kernel: 'gemv' | ('tiled', tn) | 'sk' (stream-K at tc_pick_tn(M), as the engine's batched decode)"""
    if kernel == "gemv":
        run_gemv(shim, epi, NORM_NONE, n_sm, M=M, **kw)
    elif kernel == "sk":
        run_tc(shim, epi, tc_pick_tn(M), n_sm, sk=sk_ws, M=M, **kw)
    else:
        run_tc(shim, epi, kernel[1], n_sm, M=M, **kw)


# ------------------------------------------------------------------------------------------------------------ host checks
def test_host_emulation_hand_values():
    """The float32 epilogue emulation and the float64 product against values worked out by hand."""
    # one RoPE pair: x0 = 1.5, x1 = -0.75, cos = 0.5, sin = 0.875 (all exact in bf16)
    # y0 = 1.5*0.5 + 0.75*0.875 = 0.75 + 0.65625 = 1.40625 ; y1 = -0.75*0.5 + 1.5*0.875 = -0.375 + 1.3125 = 0.9375
    y0, y1 = rope_ref(torch.tensor([1.5]), torch.tensor([-0.75]), torch.tensor([0.5]), torch.tensor([0.875]))
    assert y0.item() == 1.40625 and y1.item() == 0.9375
    # rounding points: x0 = 1 + 2^-7 (exact bf16), cos = 1 + 2^-7 -> x0*cos = 1 + 2^-6 + 2^-14 -> bf16 1 + 2^-6
    y0, _ = rope_ref(torch.tensor([1 + 2 ** -7]), torch.tensor([0.0]), torch.tensor([1 + 2 ** -7]), torch.tensor([0.0]))
    assert y0.item() == 1 + 2 ** -6
    # one SwiGLU element: g = 2, u = 3: silu(2) = 2 / (1 + e^-2) = 1.76159...; bf16 (step 2^-7) -> 1.7578125;
    # * 3 = 5.2734375 -> bf16 (step 2^-5) 5.28125
    out = epilogue_ref(EPI_SWIGLU, torch.tensor([[2.0, 3.0]]))
    assert out.float().item() == 5.28125
    # residual: bf16(acc) + resid rounded once: acc = 1 + 2^-9 -> 1; 1 + 2^-8 (resid) -> tie, stays 1 (even)
    out = epilogue_ref(EPI_RESID, torch.tensor([[1 + 2 ** -9, 0.0]]), resid=torch.tensor([[2 ** -8, 0.0]]))
    assert out.float()[0, 0].item() == 1.0
    # float64 product of dyadic inputs: [0.5, -0.25] . [0.125, 0.0625] = 0.0625 - 0.015625
    x = torch.tensor([[0.5, -0.25]], dtype=torch.bfloat16)
    W = torch.tensor([[0.125, 0.0625]], dtype=torch.bfloat16)
    assert matmul64(x, W).item() == 0.046875
    assert ulp_bf16(torch.tensor([1.0, 1.99, 0.75])).tolist() == [2 ** -7, 2 ** -7, 2 ** -8]


# ------------------------------------------------------------------------------------------------------------ GEMV
GEMV_EXACT = [  # (M, K, N, n_sm): M = 3 rides the padded 4-row tile, M 5..8 are two row tiles; at K = 28672 the tile height drops
    (1, 8, 2, "all"), (2, 120, 18, 7), (3, 1016, 130, 1), (4, 1024, 4096, "all"), (1, 1032, 130, "all"),
    (3, 4096, 32000, "all"), (4, 11008, 4096, 7), (2, 28672, 4096, "all"), (4, 28672, 18, 1), (5, 4096, 4096, "all"),
    (8, 1032, 130, 7), (6, 28672, 130, "all"), (7, 120, 2, 1),
]


@pytest.mark.parametrize("M,K,N,nsm", GEMV_EXACT)
def test_gemv_f32_exact(shim, n_sm, M, K, N, nsm):
    gen = torch.Generator(device=DEV).manual_seed(M * 7919 + K + N)
    W, x = dyadic((N, K), gen), dyadic((M, K), gen)
    out = torch.full((M, N), float("nan"), device=DEV)
    run_gemv(shim, EPI_F32, NORM_NONE, nsm_of(nsm, n_sm), W=W, x=x, N=N, K=K, ldx=K, M=M, out_f32=out, ld_out=N)
    assert_same_bits(out, matmul64(x, W).float(), f"GEMV M={M} K={K} N={N}")
    if K == 28672 and M >= 3:
        assert shim.shim_gemv_pick_bt(M, K) == 2  # 4 rows of staged activations do not fit beside the ring


@pytest.mark.parametrize("M", [3, 5, 8])
def test_gemv_row_map_and_f32_add(shim, n_sm, M):
    """row_map gathers x rows in a non-monotone order from a larger buffer (the prefill lm_head); f32_add is the optional
    fp32 addend of EPI_F32."""
    gen = torch.Generator(device=DEV).manual_seed(100 + M)
    K, N, X = 4096, 4098, 19
    W, x = dyadic((N, K), gen), dyadic((X, K), gen)
    rows = torch.randperm(X, generator=torch.Generator().manual_seed(M))[:M].int()
    add = dyadic((M, N), gen).float()
    out = torch.empty(M, N, device=DEV)
    run_gemv(shim, EPI_F32, NORM_NONE, n_sm, W=W, x=x, N=N, K=K, ldx=K, M=M, row_map=rows.to(DEV), f32_add=add, out_f32=out,
             ld_out=N)
    assert_same_bits(out, (matmul64(x, W, rows) + add.cpu().double()).float(), f"GEMV row_map M={M}")


def epilogue_inputs(epi, M, N, gen):
    kw, ref_kw = {}, {}
    if epi in (EPI_RESID, EPI_RESID2):
        kw["resid"] = ref_kw["resid"] = dyadic((M, N), gen, 2.0 ** -2)
    if epi == EPI_RESID2:
        kw["resid2"] = ref_kw["resid2"] = dyadic((M, N), gen, 2.0 ** -3)
    return kw, ref_kw


EPIS_BF16 = [EPI_F32_BF16R, EPI_BF16, EPI_RESID, EPI_RESID2, EPI_SWIGLU, EPI_GELU]


@pytest.mark.parametrize("kernel,M,K,N", [
    ("gemv", 3, 1032, 1030), ("gemv", 6, 4096, 258),
    (("tiled", 128), 70, 1376, 386), (("tiled", 16), 17, 72, 130), (("tiled", 256), 257, 1024, 254),
    ("sk", 20, 4096, 1030), ("sk", 64, 11008, 4096), ("sk", 1, 2752, 258),
])
@pytest.mark.parametrize("epi", EPIS_BF16)
def test_projection_epilogues(shim, n_sm, sk_ws, kernel, M, K, N, epi):
    """Every bf16 epilogue on an exact accumulator: bit for bit against the float32 emulation (SWIGLU / GELU: one ulp on
    at most 1 % of the elements).  EPI_RESID runs in place (out == resid), as the engine runs o_proj and down."""
    if kernel == "gemv" and epi in (EPI_F32_BF16R, EPI_SWIGLU, EPI_GELU):
        pytest.skip("the GEMV has these epilogues only behind a fused norm (test_gemv_fused_norm)")
    gen = torch.Generator(device=DEV).manual_seed(M * 31 + N + epi)
    W, x = dyadic((N, K), gen), dyadic((M, K), gen)
    kw, ref_kw = epilogue_inputs(epi, M, N, gen)
    want = epilogue_ref(epi, matmul64(x, W).float(), **ref_kw)
    ld_out = N // 2 if epi == EPI_SWIGLU else N
    if epi == EPI_F32_BF16R:
        out = torch.full((M, N), float("nan"), device=DEV)
        kw["out_f32"] = out
    elif epi == EPI_RESID:
        out = kw["resid"]  # in place
        kw["out_bf16"] = out
    else:
        out = torch.full((M, ld_out), float("nan"), device=DEV, dtype=torch.bfloat16)
        kw["out_bf16"] = out
    run_proj(shim, kernel, epi, n_sm, sk_ws, M, W=W, x=x, N=N, K=K, ldx=K, ld_out=ld_out, **kw)
    what = f"{kernel} epi={epi} M={M} K={K} N={N}"
    if epi == EPI_GELU:
        assert_gelu(out, matmul64(x, W), what)
    elif epi == EPI_SWIGLU:
        assert_within_ulp(out, want, what, 0.01)
    else:
        assert_same_bits(out, want, what)


@pytest.mark.parametrize("norm,epi,M,K", [
    (NORM_RMS, EPI_F32_BF16R, 1, 4096), (NORM_RMS, EPI_SWIGLU, 3, 5120), (NORM_RMS, EPI_F32_BF16R, 8, 1032),
    (NORM_LN, EPI_F32_BF16R, 2, 4096), (NORM_LN, EPI_GELU, 4, 8192), (NORM_LN, EPI_F32_BF16R, 6, 1016),
])
def test_gemv_fused_norm(shim, n_sm, norm, epi, M, K):
    """The GEMV's fused RMSNorm / LayerNorm prologue against the standalone norm kernel on the same rows: both reduce with
    256 threads at a stride of 2048 elements, warp sums, then 8 warps in order, so the normed activations and therefore
    the accumulators must match bit for bit.  The accumulator itself is checked against float64 within proj_bound."""
    gen = torch.Generator(device=DEV).manual_seed(norm * 1000 + M + K)
    N = 2050
    W, x = dyadic((N, K), gen), continuous((M, K), gen, 3.0)
    nw, nb = continuous((K,), gen, 0.5), continuous((K,), gen, 0.1)
    eps = 1e-5
    xn = torch.empty_like(x)
    if norm == NORM_RMS:
        launch(shim.shim_rmsnorm, _ptr(x), _ptr(nw), _ptr(xn), M, K, eps)
    else:
        launch(shim.shim_layernorm, _ptr(x), _ptr(nw), _ptr(nb), _ptr(xn), M, K, eps)
    acc = torch.empty(M, N, device=DEV)
    run_gemv(shim, EPI_F32, NORM_NONE, n_sm, W=W, x=xn, N=N, K=K, ldx=K, M=M, out_f32=acc, ld_out=N)
    assert within(acc, matmul64(xn, W), proj_bound(xn, W)), "GEMV on the normed rows vs float64"
    ld_out = N // 2 if epi == EPI_SWIGLU else N
    out = torch.empty(M, ld_out, device=DEV, dtype=torch.float32 if epi == EPI_F32_BF16R else torch.bfloat16)
    kw = dict(out_f32=out) if epi == EPI_F32_BF16R else dict(out_bf16=out)
    run_gemv(shim, epi, norm, n_sm, W=W, x=x, N=N, K=K, ldx=K, M=M, norm_w=nw, norm_b=nb, eps=eps, ld_out=ld_out, **kw)
    want = epilogue_ref(epi, acc.cpu())
    if epi == EPI_F32_BF16R:
        assert_same_bits(out, want, f"fused norm={norm} M={M} K={K}")
    elif epi == EPI_GELU:
        assert_gelu(out, acc, f"fused norm={norm} M={M} K={K}")
    else:
        assert_within_ulp(out, want, f"fused norm={norm} epi={epi} M={M} K={K}", 0.01)


# ------------------------------------------------------------------------------------------------------------ wgmma
TILED = [  # (tn, M, N, K, n_sm)
    (16, 1, 128, 64, "all"), (16, 15, 130, 72, "all"), (16, 17, 254, 1376, 7), (16, 16, 2752, 4096, "all"),
    (32, 63, 4096, 1376, "all"), (32, 65, 130, 11008, 7), (64, 64, 254, 4096, "all"), (64, 127, 2752, 72, "all"),
    (64, 1, 4096, 11008, 33), (128, 128, 4096, 4096, "all"), (128, 129, 130, 1376, "all"), (128, 255, 254, 11008, 7),
    (128, 17, 254, 72, "all"), (256, 256, 2752, 64, "all"), (256, 257, 4096, 1376, "all"), (256, 300, 128, 4096, 7),
]


@pytest.mark.parametrize("tn,M,N,K,nsm", TILED)
def test_tc_tiled_f32_exact(shim, n_sm, tn, M, N, K, nsm):
    """tc_gemm_kernel (no stream-K workspace): every token tile, N tail (TMA zero fill) and K tail."""
    gen = torch.Generator(device=DEV).manual_seed(tn * 1009 + M * 13 + N + K)
    W, x = dyadic((N, K), gen), dyadic((M, K), gen)
    out = torch.full((M, N), float("nan"), device=DEV)
    run_tc(shim, EPI_F32, tn, nsm_of(nsm, n_sm), W=W, x=x, N=N, K=K, ldx=K, M=M, out_f32=out, ld_out=N)
    assert_same_bits(out, matmul64(x, W).float(), f"tiled tn={tn} M={M} N={N} K={K}")


def sk_spans(N, K, n_sm):
    """Most CTA ranges one weight tile spans in the stream-K partition (mirror of csrc/sk_partition.h)."""
    nkb = (K + 63) // 64
    U = ((N + 127) // 128) * nkb
    G = max(1, min(U // ((nkb + 7) // 8), n_sm))
    beg = lambda b: b * U // G
    return max(sum(1 for b in range(G) if beg(b) < (t + 1) * nkb and beg(b + 1) > t * nkb) for t in range((N + 127) // 128))


LLAMA7B = dict(qkv=(12288, 4096), o=(4096, 4096), gu=(22016, 4096), down=(4096, 11008), lm=(32000, 4096))
STREAMK = [  # (M, N, K, n_sm): Llama-2-7B projections, their tensor-parallel shards, and long-K one- to three-tile matrices
    (1, *LLAMA7B["qkv"], "all"), (5, *LLAMA7B["o"], 33), (16, *LLAMA7B["gu"], "all"), (17, *LLAMA7B["down"], "all"),
    (31, *LLAMA7B["lm"], 7), (32, 6144, 4096, "all"), (33, 4096, 2048, 33), (64, 11008, 4096, "all"),
    (64, 4096, 5504, 7), (17, 16000, 4096, "all"), (33, 4096, 2752, "all"), (5, 4096, 1376, 7), (64, *LLAMA7B["down"], 33),
    (1, 128, 28672, "all"), (16, 256, 28672, "all"), (32, 384, 28608, "all"), (64, 128, 28608, 33), (5, 256, 4160, 7),
]


@pytest.mark.parametrize("M,N,K,nsm", STREAMK)
def test_tc_streamk_f32_exact(shim, n_sm, sk_ws, M, N, K, nsm):
    """tc_gemm_sk_kernel at TN 16 / 32 / 64: exact product, two launches bit-identical, every flag word zero afterwards."""
    gen = torch.Generator(device=DEV).manual_seed(M * 131 + N + K)
    W, x = dyadic((N, K), gen), dyadic((M, K), gen)
    outs = []
    for _ in range(2):
        out = torch.full((M, N), float("nan"), device=DEV)
        run_tc(shim, EPI_F32, tc_pick_tn(M), nsm_of(nsm, n_sm), sk=sk_ws, W=W, x=x, N=N, K=K, ldx=K, M=M, out_f32=out, ld_out=N)
        assert int(sk_ws[1].abs().sum()) == 0, "stream-K flags not reset"
        outs.append(out)
    assert_same_bits(outs[0], matmul64(x, W).float(), f"stream-K M={M} N={N} K={K} n_sm={nsm}")
    assert same_bits(outs[0], outs[1]), "two stream-K launches differ"


def test_streamk_cases_reach_the_partition_limits(n_sm):
    """The long-K cases above make one tile span 8 or 9 CTA ranges (the grid cap of sk_grid), the most the partition allows."""
    spans = [sk_spans(N, K, nsm_of(nsm, n_sm)) for M, N, K, nsm in STREAMK if K > 20000]
    assert max(spans) >= 9 and min(spans) >= 4, spans


def test_projections_continuous(shim, n_sm, sk_ws):
    """Ordinary bf16 data on all three projection kernels (M = 4, as a batch-4 decode): each within 2^-16 sum|w x| of
    float64, each pair within the same bound of each other; the check rejects a reference missing the last k-block."""
    gen = torch.Generator(device=DEV).manual_seed(77)
    M, N, K = 4, 4096, 4096
    W, x = continuous((N, K), gen, 0.05), continuous((M, K), gen)
    ref, bound = matmul64(x, W), proj_bound(x, W)
    outs = {}
    for kernel in ("gemv", ("tiled", 16), "sk"):
        out = torch.empty(M, N, device=DEV)
        run_proj(shim, kernel, EPI_F32, n_sm, sk_ws, M, W=W, x=x, N=N, K=K, ldx=K, out_f32=out, ld_out=N)
        err = float(((out.cpu().double() - ref).abs() / bound).max())
        print(f"continuous {kernel}: max |err| / bound = {err:.3f}")
        assert err <= 1.0, kernel
        outs[str(kernel)] = out.cpu().double()
    names = list(outs)
    for a in range(3):
        for b in range(a + 1, 3):
            assert bool(((outs[names[a]] - outs[names[b]]).abs() <= bound).all()), (names[a], names[b])
    short = matmul64(x[:, :K - 64], W[:, :K - 64])
    assert not within(outs[names[0]], short, proj_bound(x[:, :K - 64], W[:, :K - 64])), "dropped k-block not rejected"


@pytest.mark.parametrize("kernel,M,tn", [(("tiled", 256), 300, 256), ("sk", 32, 32)])
def test_tc_continuous_large(shim, n_sm, sk_ws, kernel, M, tn):
    gen = torch.Generator(device=DEV).manual_seed(M)
    N, K = (2752, 4096) if kernel != "sk" else (4096, 11008)
    W, x = continuous((N, K), gen, 0.05), continuous((M, K), gen)
    out = torch.empty(M, N, device=DEV)
    run_proj(shim, kernel, EPI_F32, n_sm, sk_ws, M, W=W, x=x, N=N, K=K, ldx=K, out_f32=out, ld_out=N)
    ref, bound = matmul64(x, W), proj_bound(x, W)
    err = float(((out.cpu().double() - ref).abs() / bound).max())
    print(f"continuous {kernel} M={M}: max |err| / bound = {err:.3f}")
    assert err <= 1.0
    assert not within(out, matmul64(x[:, :K - 64], W[:, :K - 64]), proj_bound(x[:, :K - 64], W[:, :K - 64]))


# ------------------------------------------------------------------------------------------------------------ QKV + RoPE
QKV = [  # (kernel, M, H, KVH, D, block size): GQA where KVH < H
    ("gemv", 3, 4, 2, 128, 16), ("gemv", 6, 8, 8, 64, 8),
    (("tiled", 128), 100, 8, 2, 64, 32), (("tiled", 64), 40, 4, 4, 128, 64), (("tiled", 16), 5, 8, 1, 128, 8),
    ("sk", 20, 8, 8, 128, 8), ("sk", 64, 16, 2, 64, 64), ("sk", 1, 4, 1, 128, 16),
]


@pytest.mark.parametrize("kernel,M,H,KVH,D,bs", QKV)
def test_qkv_rope_kv_append(shim, n_sm, sk_ws, kernel, M, H, KVH, D, bs):
    """EPI_QKV_ROPE: q, and k/v written into shuffled paged caches at each row's (slot, position), bit for bit; every cache
    cell outside the written (block, head, offset) cells keeps its sentinel; a position shifted by one is rejected."""
    gen = torch.Generator(device=DEV).manual_seed(M * 17 + H + D + bs)
    hgen = torch.Generator().manual_seed(M + D)
    max_pos, slots = 512, M + 3
    K, N = 1024, (H + 2 * KVH) * D
    kv = KvLayout(slots, max_pos, bs, KVH, D, hgen)
    # rows: distinct slots, positions at block edges, block interiors and the last position
    slot = torch.randperm(slots, generator=hgen)[:M].int()
    edge = torch.tensor([0, bs - 1, bs, bs + 1, max_pos - 1, 2 * bs - 1, 3 * bs])
    pos = torch.where(torch.arange(M) < len(edge), edge[torch.arange(M) % len(edge)],
                      torch.randint(0, max_pos, (M,), generator=hgen)).int()
    table, cos, sin = rope_table(max_pos + 1, D)
    W = dyadic((N, K), gen)
    kc, vc = kv.empty_cache(), kv.empty_cache()
    q = torch.full((M, H * D), float("nan"), device=DEV, dtype=torch.bfloat16)
    kw = dict(W=W, N=N, K=K, ldx=K, M=M, q_out=q, q_rows=H * D, kv_rows=KVH * D, head_dim=D, kcache=kc, vcache=vc,
              block_table=kv.bt_dev, bt_stride=kv.stride, row_slot=slot.to(DEV), row_pos=pos.to(DEV), rope_cs=table,
              block_size=bs, kvh=KVH)
    if kernel == "gemv":  # the GEMV has this epilogue only behind the fused RMSNorm: accumulator from the standalone norm
        x, nw = continuous((M, K), gen, 2.0), continuous((K,), gen, 0.5)
        xn = torch.empty_like(x)
        launch(shim.shim_rmsnorm, _ptr(x), _ptr(nw), _ptr(xn), M, K, 1e-5)
        acc = torch.empty(M, N, device=DEV)
        run_gemv(shim, EPI_F32, NORM_NONE, n_sm, W=W, x=xn, N=N, K=K, ldx=K, M=M, out_f32=acc, ld_out=N)
        acc = acc.cpu()
        run_gemv(shim, EPI_QKV_ROPE, NORM_RMS, n_sm, x=x, norm_w=nw, eps=1e-5, **kw)
    else:
        x = dyadic((M, K), gen)
        acc = matmul64(x, W).float()
        run_proj(shim, kernel, EPI_QKV_ROPE, n_sm, sk_ws, x=x, **kw)
    want_q, want_k, want_v = qkv_ref(acc, pos, slot, H, KVH, D, cos, sin, kv)
    what = f"{kernel} M={M} H={H} KVH={KVH} D={D} bs={bs}"
    assert_same_bits(q, want_q, "q " + what)
    assert_same_bits(kc, want_k, "k cache " + what)
    assert_same_bits(vc, want_v, "v cache " + what)
    shifted_q, _, _ = qkv_ref(acc, pos + 1, slot, H, KVH, D, cos, sin, kv, caches=False)
    assert not same_bits(q, shifted_q), "RoPE at position + 1 not rejected"


# ------------------------------------------------------------------------------------------------------------ attention
def attn_ref(q, K, V, scale, group):
    """q [H, D] (exact bf16 values), K / V [T, KVH, D] -> float64 [H, D].  Scores bf16(bf16(q.k) * scale) are exact."""
    H, D = q.shape
    KVH = K.shape[1]
    d = torch.einsum("kgd,tkd->kgt", q.double().view(KVH, group, D), K.double()).float()  # exact: dyadic products
    s = bf(bf(d) * np.float32(scale)).double()
    p = torch.softmax(s, dim=-1)
    return torch.einsum("kgt,tkd->kgd", p, V.double()).reshape(H, D)


def attn_bound(ref, v_max, pv_dev=None):
    """|kernel - float64| <= ulp_bf16(ref) + 2^-16 max|v| (+ 2^-8 / (1 - 2^-8) * max_i |v_i - ref| with a bf16 P).
    ulp: the final rounding to bf16 (half an ulp of the fp32 result, which may sit in the next binade up).  2^-16 max|v|:
    the fp32 online softmax — __expf (about 2 fp32 ulps) and fp32 running sums of p and p v over at most 4096 keys, whose
    relative error stays far below 2^-16.  bf16 P (prefill): each key's weight carries a relative error e_i <= 2^-8 in both
    the numerator and the normaliser, so the result moves by sum w_i e_i (v_i - ref) / sum w_i (1 + e_i)."""
    b = ulp_bf16(ref) + 2.0 ** -16 * v_max
    if pv_dev is not None:
        b = b + 2.0 ** -8 / (1 - 2.0 ** -8) * pv_dev
    return b


def make_kv_rows(ctxs, KVH, D, gen):
    return [(dyadic((c, KVH, D), gen).cpu(), continuous((c, KVH, D), gen, 0.25).clamp(-0.5, 0.5).cpu()) for c in ctxs]


def fill_cache(kv, slots, rows):
    kc, vc = kv.empty_cache().cpu(), kv.empty_cache().cpu()
    for s, (Kr, Vr) in zip(slots, rows):
        blk, off = kv.cells(torch.full((Kr.shape[0],), int(s)), torch.arange(Kr.shape[0]))
        kc[blk, :, off] = Kr.to(torch.bfloat16)
        vc[blk, :, off] = Vr.to(torch.bfloat16)
    return kc.to(DEV), vc.to(DEV)


def split_chunk(ctx, n_splits, bs):
    chunk = -(-ctx // n_splits)
    return -(-chunk // bs) * bs


DECODE = [  # (D, group, n_splits, block size): group 1 / 2 = attn_decode_kernel G1 / G2, 4 / 8 = attn_gqa_kernel G4 / G8
    (128, 1, 1, 16), (128, 1, 32, 8), (64, 1, 7, 64), (128, 2, 16, 32), (64, 2, 2, 16), (128, 2, 32, 64),
    (128, 4, 16, 16), (64, 4, 7, 8), (128, 8, 16, 64), (64, 8, 2, 32), (128, 8, 1, 8),
]


@pytest.mark.parametrize("D,group,n_splits,bs", DECODE)
def test_attn_decode(shim, D, group, n_splits, bs):
    """Split-context decode attention, one batch of 32 rows with contexts at block and split-chunk edges up to 4096."""
    gen = torch.Generator(device=DEV).manual_seed(D + group * 10 + n_splits * 100 + bs)
    hgen = torch.Generator().manual_seed(n_splits * 7 + bs)
    KVH, max_pos = 2, 4096
    H = KVH * group
    nb = n_splits * bs
    ctxs = [1, bs - 1, bs, bs + 1, 900, 4096, nb, nb + 1, nb - 1, 3 * nb + 1, 2 * nb - 1, 2, 17, 64, 65, 100, 257, 511,
            1000, 2047, 2049, 3001, 4095, 130, 33, 1024, 1025, 5 * bs + 3, 700, 1500, 63, 3]
    ctxs = [min(max(c, 1), max_pos) for c in ctxs][:32]
    M, slots = len(ctxs), len(ctxs) + 2
    kv = KvLayout(slots, max_pos, bs, KVH, D, hgen)
    slot = torch.randperm(slots, generator=hgen)[:M].int()
    rows = make_kv_rows(ctxs, KVH, D, gen)
    kc, vc = fill_cache(kv, slot.tolist(), rows)
    q = dyadic((M, H * D), gen, 2.0 ** -3)
    scale = np.float32(1.0) / np.sqrt(np.float32(D))
    gc = 8 if group % 8 == 0 else 4 if group % 4 == 0 else 2 if group % 2 == 0 else 1
    part_o = torch.zeros(M * H * n_splits * D, device=DEV)
    part_ml = torch.zeros(M * H * n_splits * 2, device=DEV)
    counters = torch.zeros(M * (H // gc), dtype=torch.int32, device=DEV)
    pos = torch.tensor([c - 1 for c in ctxs], dtype=torch.int32)
    outs = []
    for _ in range(2):
        out = torch.full((M, H * D), float("nan"), device=DEV, dtype=torch.bfloat16)
        a = _struct(ShimAttn, q=q, kcache=kc, vcache=vc, block_table=kv.bt_dev, bt_stride=kv.stride, row_slot=slot.to(DEV),
                    row_pos=pos.to(DEV), out=out, part_o=part_o, part_ml=part_ml, counters=counters, M=M, n_heads=H, kvh=KVH,
                    group=group, head_dim=D, block_size=bs, n_splits=n_splits, scale=float(scale))
        launch(shim.shim_attn_decode, C.byref(a))
        assert int(counters.abs().sum()) == 0, "split counters not reset"
        outs.append(out.cpu())
    assert same_bits(outs[0], outs[1]), "two decode-attention launches differ"
    got = outs[0].double()
    qc = q.cpu()

    def reference(keys_of):
        return torch.stack([attn_ref(qc[m].view(H, D), rows[m][0][keys_of(m)], rows[m][1][keys_of(m)], scale, group).reshape(-1)
                            for m in range(M)])

    v_max = max(float(r[1].abs().max()) for r in rows)
    ref = reference(lambda m: slice(None))
    bound = attn_bound(ref, v_max)
    err = (got - ref).abs() / bound
    print(f"decode D={D} G={group} splits={n_splits} bs={bs}: max |err| / bound = {float(err.max()):.3f}")
    worst = int(err.max(dim=1).values.argmax())
    assert bool((err <= 1).all()), f"row {worst} (ctx {ctxs[worst]}): max |err| / bound = {float(err.max()):.3f}"

    # negative controls: the same check rejects a reference that drops the last key, drops the first key of a split, or
    # counts a split twice (rows whose context is cut into several splits)
    def rejected(keys_of):
        wrong = reference(keys_of)
        return not bool(((got - wrong).abs() <= attn_bound(wrong, v_max)).all())

    def idx(m, drop=None, dup=None):
        c = ctxs[m]
        ks = [t for t in range(c) if t != drop]
        if dup is not None:
            ks += list(range(*dup))
        return torch.tensor(ks if ks else [0])

    chunks = [split_chunk(c, n_splits, bs) for c in ctxs]
    multi = [m for m in range(M) if chunks[m] < ctxs[m]]
    assert rejected(lambda m: idx(m, drop=ctxs[m] - 1 if ctxs[m] > 1 else None)), "dropped last key not rejected"
    if multi:
        assert rejected(lambda m: idx(m, drop=chunks[m] if m in multi else None)), "dropped first key of split 1 not rejected"
        assert rejected(lambda m: idx(m, dup=(0, chunks[m]) if m in multi else None)), "split counted twice not rejected"
    else:
        assert n_splits == 1


PREFILL = [  # (D, group, block size)
    (128, 1, 16), (64, 2, 8), (128, 4, 32), (64, 8, 64), (128, 8, 16),
]


@pytest.mark.parametrize("D,group,bs", PREFILL)
def test_attn_prefill(shim, D, group, bs):
    """Causal prefill attention over tiles of <= 64 consecutive rows of one sequence, several sequences per launch,
    including chunked prefills that continue an existing cache (pos0 > 0) and a sequence cut into 40 + 24-row tiles."""
    gen = torch.Generator(device=DEV).manual_seed(D * 3 + group + bs)
    hgen = torch.Generator().manual_seed(D + bs)
    KVH, max_pos = 2, 512
    H = KVH * group
    # (pos0, new rows, tile cut) per sequence; ctx = pos0 + new rows keys in the cache
    seqs = [(0, 64, [64]), (0, 1, [1]), (0, 130, [64, 64, 2]), (37, 50, [50]), (100, 64, [40, 24]), (200, 5, [5]),
            (448, 64, [64]), (63, 2, [2])]
    slots = len(seqs) + 1
    kv = KvLayout(slots, max_pos, bs, KVH, D, hgen)
    slot_of = torch.randperm(slots, generator=hgen)[:len(seqs)].tolist()
    rows = make_kv_rows([p + n for p, n, _ in seqs], KVH, D, gen)
    kc, vc = fill_cache(kv, slot_of, rows)
    row_slot, row_pos, tile_row0, tile_nrows, row_seq = [], [], [], [], []
    for si, (p0, n, cuts) in enumerate(seqs):
        r = len(row_pos)
        for c in cuts:
            tile_row0.append(r)
            tile_nrows.append(c)
            r += c
        row_slot += [slot_of[si]] * n
        row_pos += list(range(p0, p0 + n))
        row_seq += [si] * n
    M = len(row_pos)
    q = dyadic((M, H * D), gen, 2.0 ** -3)
    out = torch.full((M, H * D), float("nan"), device=DEV, dtype=torch.bfloat16)
    scale = np.float32(1.0) / np.sqrt(np.float32(D))
    i32 = lambda v: torch.tensor(v, dtype=torch.int32, device=DEV)
    a = _struct(ShimAttn, q=q, kcache=kc, vcache=vc, block_table=kv.bt_dev, bt_stride=kv.stride, row_slot=i32(row_slot),
                row_pos=i32(row_pos), tile_row0=i32(tile_row0), tile_nrows=i32(tile_nrows), out=out, M=M, n_heads=H, kvh=KVH,
                group=group, head_dim=D, block_size=bs, n_splits=1, n_tiles=len(tile_row0), scale=float(scale))
    launch(shim.shim_attn_prefill, C.byref(a))
    got, qc = out.cpu().double(), q.cpu()
    v_max = max(float(r[1].abs().max()) for r in rows)

    def check(keys_of):
        ref = torch.stack([attn_ref(qc[m].view(H, D), rows[row_seq[m]][0][keys_of(m)], rows[row_seq[m]][1][keys_of(m)],
                                    scale, group).reshape(-1) for m in range(M)])
        # per element: max over the row's keys of |v_i - ref| (heads are kv-major: head = kv head * group + g)
        dev = torch.stack([(rows[row_seq[m]][1][keys_of(m)].double()[:, :, None, :] - ref[m].view(1, KVH, group, D))
                           .abs().amax(0).reshape(-1) for m in range(M)])
        return (got - ref).abs() / attn_bound(ref, v_max, dev)

    err = check(lambda m: torch.arange(row_pos[m] + 1))
    print(f"prefill D={D} G={group} bs={bs}: max |err| / bound = {float(err.max()):.3f}")
    assert bool((err <= 1).all()), f"max |err| / bound = {float(err.max()):.3f}"
    # negative controls: drop the diagonal (last) key of every row with more than one key; count the first 64-key chunk
    # twice for rows whose context is longer than one chunk
    assert not bool((check(lambda m: torch.arange(max(row_pos[m], 1))) <= 1).all()), "dropped last key not rejected"
    twice = lambda m: torch.cat([torch.arange(row_pos[m] + 1), torch.arange(64 if row_pos[m] >= 64 else 0)])
    assert not bool((check(twice) <= 1).all()), "chunk counted twice not rejected"


# ------------------------------------------------------------------------------------------------------------ norms, argmax
@pytest.mark.parametrize("K", [256, 4096, 5120, 8192])
@pytest.mark.parametrize("kind", ["rms", "ln"])
def test_norms(shim, kind, K):
    """Standalone RMSNorm / LayerNorm against float64 statistics: within one rounding at each bf16 rounding point."""
    gen = torch.Generator(device=DEV).manual_seed(K + len(kind))
    M, eps = 5, 1e-5
    x = continuous((M, K), gen, 2.0)
    x[1] = x[1] + 3.0  # a row with a large mean (LayerNorm cancellation)
    x[2] = x[2] * 1e-2
    w, b = continuous((K,), gen, 0.5), continuous((K,), gen, 0.1)
    out = torch.empty_like(x)
    if kind == "rms":
        launch(shim.shim_rmsnorm, _ptr(x), _ptr(w), _ptr(out), M, K, eps)
    else:
        launch(shim.shim_layernorm, _ptr(x), _ptr(w), _ptr(b), _ptr(out), M, K, eps)
    xd, wd, bd = x.cpu().double(), w.cpu().double(), b.cpu().double()
    if kind == "rms":
        r = torch.rsqrt((xd * xd).mean(1, keepdim=True) + eps)
        inner = bf((xd * r).float()).double()  # HF: bf16(x * rstd) before the weight multiply
        ref = inner * wd
        # one ulp of the inner rounding (times |w|) plus the final rounding
        bound = ulp_bf16(inner) * wd.abs() + ulp_bf16(ref)
    else:
        mu = xd.mean(1, keepdim=True)
        rstd = torch.rsqrt(((xd - mu) ** 2).mean(1, keepdim=True) + eps)
        t = (xd - mu) * rstd * wd
        ref = t + bd
        # final rounding, plus the fp32 statistics (mean and variance to 2^-16 of the row's magnitude) and the fused add
        bound = ulp_bf16(ref) + 2.0 ** -16 * (t.abs() + bd.abs() + rstd * wd.abs() * xd.abs().mean(1, keepdim=True))
    err = (out.cpu().double() - ref).abs() / bound
    print(f"{kind}norm K={K}: max |err| / bound = {float(err.max()):.3f}")
    assert bool((err <= 1).all())


@pytest.mark.parametrize("V", [1008, 32000, 50272, 65024])
def test_argmax(shim, V):
    """Greedy pick: lowest index on ties within a thread, across threads and across warps; -inf entries; hist / pos_inc."""
    g = torch.Generator().manual_seed(V)
    rows = []
    rows.append(torch.randn(V, generator=g))                     # plain
    r = torch.randn(V, generator=g); r[[i for i in (1029, 2053, 3000, 500 if V < 2053 else V - 1) if i < V]] = 9.0
    rows.append(r)                                               # ties: thread 5 at 1029 and 2053, other threads and warps
    r = torch.randn(V, generator=g); r[[700, 33, 700 - 32]] = 7.0
    rows.append(r)                                               # ties across warps only, lowest not the first visited
    r = torch.full((V,), float("-inf")); r[V // 2] = -1e30; r[V - 2] = -1e30
    rows.append(r)                                               # -inf everywhere but two tied finite values
    rows.append(torch.full((V,), float("-inf")))                 # all -inf: index 0
    r = torch.randn(V, generator=g); r[V - 1] = 50.0
    rows.append(r)                                               # maximum at the last index
    logits = torch.stack(rows)
    n = logits.shape[0]
    want = torch.from_numpy(np.argmax(logits.numpy(), axis=1)).int()
    tok = torch.full((n,), -1, dtype=torch.int32, device=DEV)
    hist = torch.full((3 * n,), -1, dtype=torch.int32, device=DEV)
    step = torch.tensor([2], dtype=torch.int32, device=DEV)
    pos = torch.arange(n, dtype=torch.int32, device=DEV) * 10
    launch(shim.shim_argmax, _ptr(logits.to(DEV)), V, n, _ptr(tok), _ptr(hist), _ptr(step), _ptr(pos))
    assert tok.cpu().tolist() == want.tolist()
    assert hist.cpu().tolist() == [-1] * (2 * n) + want.tolist()
    assert pos.cpu().tolist() == [10 * i + 1 for i in range(n)]
    tok2 = torch.full((n,), -1, dtype=torch.int32, device=DEV)
    launch(shim.shim_argmax, _ptr(logits.to(DEV)), V, n, _ptr(tok2), None, None, None)
    assert tok2.cpu().tolist() == want.tolist()
