"""Kernel-level tests of the persistent decode kernel (csrc/mega.cu decode_mega_kernel), launched by itself through
tests/kernel_shim.cpp::shim_decode_mega with the launch geometry of mega_geometry, the function the engine uses.

(a) Teacher-forced bit identity.  The kernel's projections share the single GEMV's consumer loop (gemv_core.cuh mma_chunk,
    1024-wide k chunks, the warp-order sum of the 8 k slices), its epilogues (epilogue.cuh) and its RMSNorm reduction
    (256 threads at a stride of 2048, 8 warps in order), and a pass's arithmetic does not depend on which CTA claims it.
    So every phase must equal shim_gemv run on the kernel's own observed input, bit for bit:
        q, K/V append   = GEMV(RMSNorm ln1, QKV_ROPE) on embed[row_tok]
        h_mid           = GEMV(RESID) of the observed attn onto embed[row_tok]   (seen as h of a launch with wdown = 0,
                                                                                  since bf16(0 + h_mid) = h_mid)
        act             = GEMV(RMSNorm ln2, SWIGLU) on h_mid
        h               = GEMV(RESID) of the observed act onto h_mid
        logits          = GEMV(RMSNorm final_norm, F32_BF16R) on h
        row_tok, hist, row_pos, step, fwd_counter = host argmax of the observed logits (lowest index wins), + 1
    test_kernels_gpu.py pins those GEMV paths to float64, so this chain pins the persistent kernel to float64 too.
(b) An exact float64 anchor that does not go through the GEMV: embedding rows +-2^-2 make the normed row exactly +-ln1,
    ln1 / wqkv / cached keys are small dyadic values and RoPE turns by quarter turns, so q and the appended K/V equal
    qkv_ref bit for bit and the attention scores are exact; attn is then within attn_bound of float64 attention.  Each
    toleranced check is paired with negative controls that must be rejected: the key this step appended dropped, the first
    key of a split dropped, a split counted twice.
(c) One L-layer launch equals L chained single-layer launches (ring, claim counters and end markers across matrices
    and layers).
(d) Barrier words and attention counters are zero after every launch; repeated launches are bit-identical; q and the
    K/V append do not depend on the grid size; greedy ties go to the lower index.

Every output buffer holds 4 rows filled with NaN (int buffers: a sentinel) before each launch, so rows at M and above must
keep it, and every KV-cache cell holds either the row's context or SENTINEL.  The kernel is cooperative and spin-waits on
its grid barrier: no launch asks for more CTAs than the device has SMs, and every launch is synchronised.
"""
import ctypes as C
import types
import zlib

import numpy as np
import pytest
import torch

from test_kernels_gpu import (DEV, EPI_F32_BF16R, EPI_QKV_ROPE, EPI_RESID, EPI_SWIGLU, NORM_NONE, NORM_RMS, SENTINEL, KvLayout,
                              _struct, abs_matmul64, assert_same_bits, attn_bound, attn_ref, continuous, dyadic, matmul64,
                              qkv_ref, rope_table, run_gemv, same_bits, shim)  # noqa: F401  (shim: the fixture)

pytestmark = pytest.mark.gpu

MG_CW = 8            # mega.cu: consumer warps per CTA
MG_ATT_TILE = 32     # mega.cu: tokens per staged tile of the CTA-tile attention
EPS = 1e-5
INVALID_VALUE = 1    # cudaErrorInvalidValue
FORM = {(0, 0): "per-warp", (1, 0): "coop", (0, 1): "cta-tile"}


class ShimMega(C.Structure):
    _fields_ = ([(n, C.c_void_p) for n in ("layers", "embed", "lm_head", "final_norm", "row_slot", "block_table", "rope_cs",
                                           "h", "q", "attn", "act", "logits", "row_tok", "row_pos", "part_o", "part_ml",
                                           "counters", "hist", "step", "fwd_counter", "grid_bar")]
                + [(n, C.c_int) for n in ("n_layers", "hidden", "n_heads", "kvh", "head_dim", "inter", "vocab", "M",
                                          "bt_stride", "block_size", "max_seq", "attn_tile")]
                + [("eps", C.c_float)])


GEOM_FIELDS = ("attn_g", "k_max", "max_chunks", "bt", "n_stages", "attn_coop", "attn_cta_tile", "part_o", "part_ml", "counters",
               "bar_words")


@pytest.fixture(scope="module")
def mshim(shim):
    shim.shim_decode_mega.argtypes = [C.POINTER(ShimMega), C.c_int]
    shim.shim_mega_geometry.argtypes = [C.POINTER(ShimMega), C.POINTER(C.c_longlong)]
    shim.shim_mega_geometry.restype = None
    return shim


@pytest.fixture(scope="module")
def n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------------------ model, step
def small_ints(shape, gen, r, scale):
    return (torch.randint(-r, r + 1, shape, generator=gen, device=DEV, dtype=torch.int32).float() * scale).to(torch.bfloat16)


def norm_weight(n, gen):
    return (1.0 + 0.1 * torch.randn(n, generator=gen, device=DEV)).to(torch.bfloat16)


class Model:
    """One model shard's weights.  exact: embedding rows +-2^-2, ln1 in {0, +-1, +-2} x 2^-2 and wqkv in {0, +-1, +-2} x 2^-4,
    so the QKV accumulator is a multiple of 2^-6 summed exactly (everything after attention stays continuous)."""

    def __init__(self, hidden, H, KVH, D, inter, vocab, L, seed, exact):
        self.hidden, self.H, self.KVH, self.D, self.inter, self.vocab, self.L, self.exact = hidden, H, KVH, D, inter, vocab, L, exact
        self.q_rows, self.kv_rows = H * D, KVH * D
        gen = torch.Generator(device=DEV).manual_seed(seed)
        n_qkv = self.q_rows + 2 * self.kv_rows
        self.layers = []
        for _ in range(L):
            if exact:
                ln1, wqkv = small_ints((hidden,), gen, 2, 2.0 ** -2), small_ints((n_qkv, hidden), gen, 2, 2.0 ** -4)
            else:
                ln1, wqkv = norm_weight(hidden, gen), continuous((n_qkv, hidden), gen, hidden ** -0.5)
            self.layers.append(types.SimpleNamespace(
                wqkv=wqkv, wo=continuous((hidden, self.q_rows), gen, self.q_rows ** -0.5),
                wgu=continuous((2 * inter, hidden), gen, hidden ** -0.5), wdown=continuous((hidden, inter), gen, inter ** -0.5),
                ln1=ln1, ln2=norm_weight(hidden, gen)))
        if exact:
            sign = torch.randint(0, 2, (vocab, hidden), generator=gen, device=DEV, dtype=torch.int32).float() * 2 - 1
            self.embed = (sign * 0.25).to(torch.bfloat16)
        else:
            self.embed = continuous((vocab, hidden), gen, 1.0)
        self.lm_head = continuous((vocab, hidden), gen, hidden ** -0.5)
        self.final_norm = norm_weight(hidden, gen)
        self.zero_down = torch.zeros(hidden, inter, dtype=torch.bfloat16, device=DEV)


def quarter_turns(max_pos, D, seed):
    """RoPE table of quarter turns, (cos, sin) in {(1,0), (0,1), (-1,0), (0,-1)} pseudo-random per (position, j): exact,
    yet a position or pair mix-up still changes the result.  Returns (device table, cos, sin) like rope_table."""
    turn = torch.randint(0, 4, (max_pos, D // 2), generator=torch.Generator().manual_seed(seed))
    c, s = torch.tensor([1.0, 0.0, -1.0, 0.0])[turn], torch.tensor([0.0, 1.0, 0.0, -1.0])[turn]
    bits = lambda t: t.to(torch.bfloat16).view(torch.int16).numpy().astype(np.uint16).astype(np.uint32)
    packed = (bits(c) | (bits(s) << 16)).view(np.int32)
    return torch.from_numpy(packed.copy()).to(DEV), c, s


class Step:
    """Inputs of one decode step: M rows with distinct slots and tokens at positions `pos`, a shuffled paged cache per layer
    holding each row's context (keys dyadic when the model is exact) and SENTINEL in every other cell."""

    def __init__(self, model, pos, bs, max_seq, seed, rope):
        hgen = torch.Generator().manual_seed(seed)
        gen = torch.Generator(device=DEV).manual_seed(seed)
        self.M, self.bs, self.max_seq = len(pos), bs, max_seq
        self.pos = torch.tensor(pos, dtype=torch.int32)
        slots = self.M + 2
        self.kv = KvLayout(slots, max_seq, bs, model.KVH, model.D, hgen)
        self.slot = torch.randperm(slots, generator=hgen)[:self.M].int()
        self.tok = torch.randperm(model.vocab, generator=hgen)[:self.M].int()
        self.table, self.cos, self.sin = rope
        valid = torch.zeros(self.kv.n_blocks, bs, dtype=torch.bool)
        for m in range(self.M):
            blk, off = self.kv.cells(int(self.slot[m]), torch.arange(int(self.pos[m])))
            valid[blk, off] = True
        mask = valid[:, None, :, None].to(DEV)
        shape = (self.kv.n_blocks, model.KVH, bs, model.D)
        sent = torch.tensor(SENTINEL, dtype=torch.int16, device=DEV)
        fill = lambda t: torch.where(mask, t.view(torch.int16), sent).view(torch.bfloat16)
        self.caches = []
        for _ in range(model.L):
            k = dyadic(shape, gen) if model.exact else continuous(shape, gen, 1.0)
            self.caches.append((fill(k), fill(continuous(shape, gen, 0.25).clamp(-0.5, 0.5))))

    def context(self, cache, m):
        """[pos_m, KVH, D] of row m's cached context (CPU)"""
        blk, off = self.kv.cells(int(self.slot[m]), torch.arange(int(self.pos[m])))
        return cache.cpu()[blk, :, off]


def i32(v):
    return torch.tensor(v, dtype=torch.int32, device=DEV)


def outputs(model, st, s0=2, f0=5):
    """Fresh output and state buffers for one launch, 4 rows each, NaN / sentinel filled; caches copied from the step."""
    nan = lambda n, dt=torch.bfloat16: torch.full((4, n), float("nan"), device=DEV, dtype=dt)
    pad = lambda t, v: t.tolist() + [v] * (4 - st.M)
    return types.SimpleNamespace(
        h=nan(model.hidden), q=nan(model.q_rows), attn=nan(model.q_rows), act=nan(model.inter),
        logits=nan(model.vocab, torch.float32), row_tok=i32(pad(st.tok, -7)), row_pos=i32(pad(st.pos, -7)),
        row_slot=i32(pad(st.slot, 0)), step=i32([s0]), fwd=i32([f0]), hist=i32([-1] * 32), s0=s0, f0=f0,
        caches=[(k.clone(), v.clone()) for k, v in st.caches])


def layer_table(layers, caches, zero_down=None):
    ptrs = [[w.wqkv.data_ptr(), w.wo.data_ptr(), w.wgu.data_ptr(), (zero_down if zero_down is not None else w.wdown).data_ptr(),
             w.ln1.data_ptr(), w.ln2.data_ptr(), k.data_ptr(), v.data_ptr()] for w, (k, v) in zip(layers, caches)]
    return torch.tensor(ptrs, dtype=torch.int64, device=DEV)


def mega_struct(model, M, max_seq, attn_tile, st=None, o=None, ws=None, table=None, layers=None, embed=None):
    kw = dict(n_layers=len(layers) if layers is not None else model.L, hidden=model.hidden, n_heads=model.H, kvh=model.KVH,
              head_dim=model.D, inter=model.inter, vocab=model.vocab, M=M, max_seq=max_seq, attn_tile=attn_tile, eps=EPS)
    if st is not None:
        kw.update(layers=table, embed=model.embed if embed is None else embed, lm_head=model.lm_head, final_norm=model.final_norm,
                  row_slot=o.row_slot, block_table=st.kv.bt_dev, rope_cs=st.table, h=o.h, q=o.q, attn=o.attn, act=o.act,
                  logits=o.logits, row_tok=o.row_tok, row_pos=o.row_pos, part_o=ws.part_o, part_ml=ws.part_ml,
                  counters=ws.counters, hist=o.hist, step=o.step, fwd_counter=o.fwd, grid_bar=ws.bar, bt_stride=st.kv.stride,
                  block_size=st.bs)
    return _struct(ShimMega, **kw)


def geometry(mshim, model, M, max_seq, attn_tile):
    out = (C.c_longlong * len(GEOM_FIELDS))()
    mshim.shim_mega_geometry(C.byref(mega_struct(model, M, max_seq, attn_tile)), out)
    g = types.SimpleNamespace(**dict(zip(GEOM_FIELDS, out)))
    g.form = FORM[(g.attn_coop, g.attn_cta_tile)]
    return g


def workspace(geo):
    """Attention partials (NaN: the kernel writes before it reads), merge counters and barrier words (zero), sized by the
    shared geometry."""
    return types.SimpleNamespace(part_o=torch.full((geo.part_o,), float("nan"), device=DEV),
                                 part_ml=torch.full((geo.part_ml,), float("nan"), device=DEV),
                                 counters=torch.zeros(geo.counters, dtype=torch.int32, device=DEV),
                                 bar=torch.zeros(geo.bar_words, dtype=torch.int32, device=DEV))


def run_mega(mshim, model, st, o, ws, n, max_seq, attn_tile, layers=None, zero_down=False, embed=None):
    """One launch on `n` CTAs; asserts success and that the kernel left its barrier words and merge counters at zero."""
    layers = model.layers if layers is None else layers
    table = layer_table(layers, o.caches, model.zero_down if zero_down else None)
    s = mega_struct(model, st.M, max_seq, attn_tile, st, o, ws, table, layers, embed)
    torch.cuda.synchronize()
    rc = mshim.shim_decode_mega(C.byref(s), n)
    torch.cuda.synchronize()
    assert rc == 0, f"shim_decode_mega returned {rc}"
    assert int(ws.bar.abs().sum()) == 0, "grid_bar words not zero after the launch"
    assert int(ws.counters.abs().sum()) == 0, "attention merge counters not zero after the launch"
    return o


# ------------------------------------------------------------------------------------------------------------ checks
def nan_rows(t, M):
    return bool(torch.isnan(t[M:].float()).all())


def check_chain(shim, n_sm, model, st, o, oz, what):
    """(a): o from the launch with the real wdown, oz from the same state with wdown = 0 (single layer)."""
    M, w = st.M, model.layers[0]
    for name in ("h", "q", "attn", "act", "logits"):
        assert nan_rows(getattr(o, name), M) and nan_rows(getattr(oz, name), M), f"{what}: {name} rows >= M written"
    for name in ("q", "attn", "act"):
        assert_same_bits(getattr(oz, name), getattr(o, name), f"{what}: {name} with wdown = 0")
    for c in range(2):
        assert_same_bits(oz.caches[0][c], o.caches[0][c], f"{what}: KV cache with wdown = 0")
    h0 = model.embed[st.tok.long().to(DEV)]
    # q and K/V append
    q_ref = torch.full((M, model.q_rows), float("nan"), device=DEV, dtype=torch.bfloat16)
    kc, vc = st.caches[0][0].clone(), st.caches[0][1].clone()
    run_gemv(shim, EPI_QKV_ROPE, NORM_RMS, n_sm, W=w.wqkv, x=h0, N=model.q_rows + 2 * model.kv_rows, K=model.hidden,
             ldx=model.hidden, M=M, norm_w=w.ln1, eps=EPS, q_out=q_ref, q_rows=model.q_rows, kv_rows=model.kv_rows,
             head_dim=model.D, kcache=kc, vcache=vc, block_table=st.kv.bt_dev, bt_stride=st.kv.stride,
             row_slot=i32(st.slot.tolist()), row_pos=i32(st.pos.tolist()), rope_cs=st.table, block_size=st.bs, kvh=model.KVH)
    assert_same_bits(o.q[:M], q_ref, f"{what}: q")
    assert_same_bits(o.caches[0][0], kc, f"{what}: K cache")
    assert_same_bits(o.caches[0][1], vc, f"{what}: V cache")
    # O projection + residual
    h_mid = h0.clone()
    run_gemv(shim, EPI_RESID, NORM_NONE, n_sm, W=w.wo, x=o.attn[:M].contiguous(), N=model.hidden, K=model.q_rows,
             ldx=model.q_rows, M=M, out_bf16=h_mid, resid=h_mid, ld_out=model.hidden)
    assert_same_bits(oz.h[:M], h_mid, f"{what}: h after O + residual")
    # RMSNorm + gate/up + SwiGLU
    act = torch.full((M, model.inter), float("nan"), device=DEV, dtype=torch.bfloat16)
    run_gemv(shim, EPI_SWIGLU, NORM_RMS, n_sm, W=w.wgu, x=oz.h[:M].contiguous(), N=2 * model.inter, K=model.hidden,
             ldx=model.hidden, M=M, norm_w=w.ln2, eps=EPS, out_bf16=act, ld_out=model.inter)
    assert_same_bits(o.act[:M], act, f"{what}: act")
    # down + residual
    h = oz.h[:M].clone()
    run_gemv(shim, EPI_RESID, NORM_NONE, n_sm, W=w.wdown, x=o.act[:M].contiguous(), N=model.hidden, K=model.inter,
             ldx=model.inter, M=M, out_bf16=h, resid=h, ld_out=model.hidden)
    assert_same_bits(o.h[:M], h, f"{what}: h after down + residual")
    check_head(shim, n_sm, model, st, o, what)


def check_head(shim, n_sm, model, st, o, what):
    """final RMSNorm + lm_head on the observed h, and the greedy pick on the observed logits"""
    M = st.M
    lg = torch.full((M, model.vocab), float("nan"), device=DEV)
    run_gemv(shim, EPI_F32_BF16R, NORM_RMS, n_sm, W=model.lm_head, x=o.h[:M].contiguous(), N=model.vocab, K=model.hidden,
             ldx=model.hidden, M=M, norm_w=model.final_norm, eps=EPS, out_f32=lg, ld_out=model.vocab)
    assert_same_bits(o.logits[:M], lg, f"{what}: logits")
    want = np.argmax(o.logits[:M].cpu().numpy(), axis=1).tolist()  # first maximum: the lowest index wins ties
    assert o.row_tok.cpu().tolist() == want + [-7] * (4 - M), f"{what}: row_tok"
    hist = [-1] * 32
    hist[(o.s0 + 1) * M:(o.s0 + 2) * M] = want
    assert o.hist.cpu().tolist() == hist, f"{what}: hist"
    assert o.row_pos.cpu().tolist() == [p + 1 for p in st.pos.tolist()] + [-7] * (4 - M), f"{what}: row_pos"
    assert int(o.step) == o.s0 + 1 and int(o.fwd) == o.f0 + 1, f"{what}: step / fwd_counter"


def same_outputs(a, b, what):
    for name in ("h", "q", "attn", "act", "logits", "row_tok", "row_pos", "hist", "step", "fwd"):
        assert same_bits(getattr(a, name), getattr(b, name)), f"{what}: {name} differs between the two launches"
    for (ka, va), (kb, vb) in zip(a.caches, b.caches):
        assert same_bits(ka, kb) and same_bits(va, vb), f"{what}: KV caches differ between the two launches"


def split_len(form, ctx, geo, model, M, n_ctas):
    """Keys per context split of the attention form (mirror of mega.cu: the per-warp chunk, the coop split rounded to
    whole RPW-token groups per warp, the CTA-tile split rounded to 32-token tiles)."""
    rpw = 32 // (model.D // 8)
    if form == "per-warp":
        return rpw * (8 if geo.attn_g <= 2 else 2)
    want, unit = split_want(form, geo, model, M, n_ctas), MG_CW * rpw if form == "coop" else MG_ATT_TILE
    return -(-(-(-ctx // want)) // unit) * unit


def split_want(form, geo, model, M, n_ctas):
    """Splits per (row, head unit) the CTA-level forms aim for: enough units to fill the grid, capped (mega.cu)."""
    want = n_ctas // max(1, M * (model.H // geo.attn_g))
    return max(1, min(want, min(8, geo.max_chunks) if form == "coop" else geo.max_chunks))


def check_exact(model, st, o, geo, n_ctas, what, stats):
    """(b): q and the appended K/V against qkv_ref, attn against float64 attention, with the negative controls."""
    M, H, KVH, D = st.M, model.H, model.KVH, model.D
    w = model.layers[0]
    x = model.embed[st.tok.long().to(DEV)].cpu().double()
    assert bool((x.abs() == 0.25).all())
    r = 0.25 / np.sqrt(0.0625 + EPS)  # x * rstd of an all-+-2^-2 row: rounds to +-1 in bf16 when within 2^-9 of 1
    assert abs(1 - r) < 2.0 ** -9 - 2.0 ** -20
    xn = (torch.sign(x) * w.ln1.cpu().double()).to(torch.bfloat16)
    # exactness: the QKV accumulator sits on the grid 2^-6 with sum |terms| far below 2^24 grid steps
    assert float(abs_matmul64(xn, w.wqkv).max()) < 2.0 ** 24 * 2.0 ** -6
    acc = matmul64(xn, w.wqkv).float()
    want_q, want_k, want_v = qkv_ref(acc, st.pos, st.slot, H, KVH, D, st.cos, st.sin, st.kv)
    blk, off = st.kv.cells(st.slot, st.pos)
    kc, vc = st.caches[0][0].cpu(), st.caches[0][1].cpu()
    kc[blk, :, off], vc[blk, :, off] = want_k[blk, :, off], want_v[blk, :, off]
    assert_same_bits(o.q[:M], want_q, f"{what}: q vs float64")
    assert_same_bits(o.caches[0][0], kc, f"{what}: K cache vs float64")
    assert_same_bits(o.caches[0][1], vc, f"{what}: V cache vs float64")
    scale = np.float32(1.0) / np.sqrt(np.float32(D))
    q = o.q[:M].cpu()
    got = o.attn[:M].cpu().double()
    keys = [torch.cat([st.context(kc, m), kc[blk[m], :, off[m]][None]]) for m in range(M)]
    vals = [torch.cat([st.context(vc, m), vc[blk[m], :, off[m]][None]]) for m in range(M)]
    for m in range(M):  # exact scores: q and K on the grid 2^-6, sum |q k| below 2^24 grid steps
        qi, ki = q[m].double().view(KVH, H // KVH, D) * 64, keys[m].double() * 64
        assert bool((qi == qi.round()).all()) and bool((ki == ki.round()).all())
        assert float(torch.einsum("kgd,tkd->kgt", qi.abs(), ki.abs()).max()) < 2.0 ** 24
    v_max = max(float(v.abs().max()) for v in vals)

    def err_of(keys_of):
        ref = torch.stack([attn_ref(q[m].view(H, D), keys[m][keys_of(m)], vals[m][keys_of(m)], scale, H // KVH).reshape(-1)
                           for m in range(M)])
        return (got - ref).abs() / attn_bound(ref, v_max)

    err = float(err_of(lambda m: slice(None)).max())
    stats.append(err)
    assert err <= 1.0, f"{what}: attn max |err| / bound = {err:.3f}"
    ctx = [int(p) + 1 for p in st.pos]
    sl = [split_len(geo.form, c, geo, model, M, n_ctas) for c in ctx]
    rejected = lambda keys_of: not bool((err_of(keys_of) <= 1).all())
    keep = lambda m, drop=None, dup=None: torch.tensor([t for t in range(ctx[m]) if t != drop] + (list(range(dup)) if dup else []))
    if max(ctx) > 1:  # the key this step appended
        assert rejected(lambda m: keep(m, drop=ctx[m] - 1 if ctx[m] > 1 else None)), f"{what}: dropped last key not rejected"
        stats.controls["last key"] += 1
    multi = [m for m in range(M) if sl[m] < ctx[m]]
    if multi:
        assert rejected(lambda m: keep(m, drop=sl[m] if m in multi else None)), f"{what}: dropped first key of split 1 not rejected"
        assert rejected(lambda m: keep(m, dup=sl[m] if m in multi else None)), f"{what}: split counted twice not rejected"
        stats.controls["split"] += 1


class Stats(list):
    def __init__(self):
        super().__init__()
        self.controls = {"last key": 0, "split": 0}


# ------------------------------------------------------------------------------------------------------------ coverage
# (id, hidden, H, KVH, D, inter, vocab, M, block size, mega_attn_tile, grid, attention form the engine's rule selects)
#   hidden 1032: a last k chunk 8 wide, O / down with P = 516 pairs; hidden 1544: a last chunk of 520; inter 688: down is
#   one partial chunk; inter 11008 / 13824: tails of 768 / 512; vocab 14: an LM head of 7 pairs.  At the full grid the small
#   matrices sit below 2 x MG_TAIL_PAIRS x n_sm pairs (claim_range's all-tail branch); grids of 1 / 4 / 7 CTAs put them
#   mostly in full passes with a clipped last tail pass.
SMALL = [
    ("d128g1-warp", 1032, 8, 8, 128, 688, 14, 1, 16, 1, "all", "per-warp"),
    ("d128g1-coop", 1544, 8, 8, 128, 1376, 64, 2, 32, 1, "all", "coop"),
    ("d64g1-warp", 1032, 16, 16, 64, 688, 130, 3, 8, 0, 7, "per-warp"),
    ("d64g1-coop", 1032, 16, 16, 64, 688, 130, 2, 64, 1, 4, "coop"),
    ("d128g2-warp", 1032, 8, 4, 128, 688, 14, 4, 8, 0, 7, "per-warp"),
    ("d128g2-coop", 1032, 8, 4, 128, 1376, 130, 3, 16, 1, "all", "coop"),
    ("d64g2-warp", 1032, 16, 8, 64, 688, 64, 1, 16, 1, 1, "per-warp"),
    ("d64g2-coop", 1032, 16, 8, 64, 688, 130, 3, 32, 1, "all", "coop"),
    ("d128g4-coop", 1032, 8, 2, 128, 11008, 130, 1, 64, 1, "all", "coop"),
    ("d128g4-warp", 1032, 8, 2, 128, 688, 14, 2, 8, 1, 4, "per-warp"),
    ("d64g4-warp", 1032, 16, 4, 64, 688, 64, 1, 32, 1, "all", "per-warp"),
    ("d64g4-coop", 1544, 16, 4, 64, 688, 130, 3, 16, 1, "all", "coop"),
    ("d128g8-warp", 1032, 16, 2, 128, 688, 130, 1, 16, 1, "all", "per-warp"),
    ("d128g16-cta", 1032, 32, 2, 128, 688, 130, 2, 32, 1, "all", "cta-tile"),
    ("d64g8-cta", 1032, 16, 2, 64, 688, 130, 4, 64, 1, 33, "cta-tile"),
    ("d64g8-warp", 1032, 16, 2, 64, 688, 64, 2, 8, 1, "all", "per-warp"),
    ("d128g1-inter13824", 1032, 8, 8, 128, 13824, 14, 1, 32, 1, 4, "coop"),
]
REAL = [  # one layer of the Llama-2 shapes
    ("7b-m1", 4096, 32, 32, 128, 11008, 32000, 1, 16, 1, "all", "coop"),
    ("7b-m4", 4096, 32, 32, 128, 11008, 32000, 4, 16, 1, "all", "coop"),
    ("13b-m1", 5120, 40, 40, 128, 13824, 32000, 1, 16, 1, "all", "coop"),
    ("70b-m1", 8192, 64, 8, 128, 28672, 32000, 1, 16, 1, "all", "cta-tile"),
    ("70b-m2", 8192, 64, 8, 128, 28672, 32000, 2, 16, 1, "all", "cta-tile"),
]
MAX_SEQ = 1024


def grid_of(kind, n_sm):
    return n_sm if kind == "all" else min(kind, n_sm)


def pos_sets(M, bs, unit, max_seq, seed, limit=None):
    """Ragged rows at pos 0 (one key: the one just appended), block edges, split edges and max_seq - 1."""
    edges = [0, bs - 1, bs, unit - 1, unit, 2 * unit - 1, 2 * unit, 3 * unit + 1, max_seq - 1, 5 * unit // 2]
    seen = []
    for e in edges:
        e = min(max(e, 0), max_seq - 1)
        if e not in seen:
            seen.append(e)
    g = torch.Generator().manual_seed(seed)
    sets = []
    for i in range(0, len(seen), M):
        s = seen[i:i + M]
        while len(s) < M:
            r = int(torch.randint(0, max_seq, (1,), generator=g))
            if r not in s:
                s.append(r)
        sets.append(s)
    return sets[:limit] if limit else sets


def run_case(mshim, n_sm, case, exact, max_seq, limit=None):
    name, hidden, H, KVH, D, inter, vocab, M, bs, tile, grid, form = case
    seed = zlib.crc32(name.encode()) % 100000 + (7 if exact else 0)
    model = Model(hidden, H, KVH, D, inter, vocab, 1, seed, exact)
    geo = geometry(mshim, model, M, max_seq, tile)
    assert geo.form == form, f"{name}: the engine's rule selects {geo.form}, the case expects {form}"
    assert geo.n_stages >= 2
    n = grid_of(grid, n_sm)
    ws = workspace(geo)
    rope = quarter_turns(max_seq + 1, D, seed) if exact else rope_table(max_seq + 1, D)
    # context lengths at which the split length steps: per-warp chunks; `want` splits of whole warp groups / tiles
    unit = split_len(form, 1, geo, model, M, n) * (1 if form == "per-warp" else split_want(form, geo, model, M, n))
    stats = Stats()
    for i, pos in enumerate(pos_sets(M, bs, unit, max_seq, seed, limit)):
        st = Step(model, pos, bs, max_seq, seed + i, rope)
        what = f"{name} {'exact' if exact else 'continuous'} pos={pos} n_ctas={n} ({form}, attn_g {geo.attn_g})"
        o = run_mega(mshim, model, st, outputs(model, st), ws, n, max_seq, tile)
        o2 = run_mega(mshim, model, st, outputs(model, st), ws, n, max_seq, tile)
        same_outputs(o, o2, what)
        oz = run_mega(mshim, model, st, outputs(model, st), ws, n, max_seq, tile, zero_down=True)
        check_chain(mshim, n_sm, model, st, o, oz, what)
        if exact:
            check_exact(model, st, o, geo, n, what, stats)
    if exact:
        print(f"{name}: attn max |err| / bound = {max(stats):.3f} over {len(stats)} steps; controls rejected: {stats.controls}")
        assert stats.controls["last key"] > 0, f"{name}: the dropped-last-key control never ran"
        # grids too small for two units per (row, head unit) leave the CTA-level forms one split: the direct-write path
        if split_len(form, max_seq, geo, model, M, n) < max_seq:
            assert stats.controls["split"] > 0, f"{name}: the split controls never ran"


@pytest.mark.parametrize("exact", [False, True], ids=["continuous", "exact"])
@pytest.mark.parametrize("case", SMALL, ids=[c[0] for c in SMALL])
def test_mega_step(mshim, n_sm, case, exact):
    """(a) for every case, (b) for the exact data; two launches bit-identical; sentinels kept."""
    run_case(mshim, n_sm, case, exact, MAX_SEQ)


@pytest.mark.parametrize("case", REAL, ids=[c[0] for c in REAL])
def test_mega_step_llama2_shapes(mshim, n_sm, case):
    run_case(mshim, n_sm, case, False, 2048, limit=2)


def test_mega_70b_batch4_refused(mshim):
    """A Llama-2-70B layer at batch 4 does not fit shared memory: the shim refuses without launching."""
    model = types.SimpleNamespace(hidden=8192, H=64, KVH=8, D=128, inter=28672, vocab=32000, L=1, q_rows=8192)
    geo = geometry(mshim, model, 4, 2048, 1)
    assert geo.n_stages == 0 and geo.bt == 4
    assert geometry(mshim, model, 2, 2048, 1).n_stages > 0
    h = torch.full((4, 8192), float("nan"), device=DEV, dtype=torch.bfloat16)
    tok, bar = i32([3, 4, 5, 6]), torch.zeros(geo.bar_words, dtype=torch.int32, device=DEV)
    s = mega_struct(model, 4, 2048, 1)
    s.h, s.row_tok, s.grid_bar = h.data_ptr(), tok.data_ptr(), bar.data_ptr()
    torch.cuda.synchronize()
    assert mshim.shim_decode_mega(C.byref(s), 1) == INVALID_VALUE
    torch.cuda.synchronize()
    assert nan_rows(h, 0) and tok.cpu().tolist() == [3, 4, 5, 6] and int(bar.abs().sum()) == 0


def test_mega_fewer_ctas_than_rows_refused(mshim, n_sm):
    """The greedy pick runs row m on CTA m, so a grid smaller than the batch must be refused before anything is written."""
    case = SMALL[4]  # d128g2-warp, M = 4
    model = Model(*case[1:7], 1, 11, False)
    geo = geometry(mshim, model, 4, MAX_SEQ, 0)
    ws = workspace(geo)
    st = Step(model, [0, 9, 100, 31], 8, MAX_SEQ, 11, rope_table(MAX_SEQ + 1, model.D))
    o = outputs(model, st)
    s = mega_struct(model, 4, MAX_SEQ, 0, st, o, ws, layer_table(model.layers, o.caches))
    torch.cuda.synchronize()
    assert mshim.shim_decode_mega(C.byref(s), 3) == INVALID_VALUE
    torch.cuda.synchronize()
    for name in ("h", "q", "attn", "act", "logits"):
        assert nan_rows(getattr(o, name), 0), f"{name} written"
    assert o.row_tok.cpu().tolist() == st.tok.tolist() and o.row_pos.cpu().tolist() == st.pos.tolist()
    assert o.hist.cpu().tolist() == [-1] * 32 and int(o.step) == 2 and int(o.fwd) == 5
    for (k, v), (k0, v0) in zip(o.caches, st.caches):
        assert same_bits(k, k0) and same_bits(v, v0)
    assert int(ws.bar.abs().sum()) == 0 and int(ws.counters.abs().sum()) == 0


@pytest.mark.parametrize("case", [SMALL[0], SMALL[5], SMALL[14]], ids=["per-warp-m1", "coop-m3", "cta-tile-m4"])
def test_mega_grid_sizes(mshim, n_sm, case):
    """q and the K/V append are bit-identical at every grid size (claims never change the arithmetic); attention and what
    follows change with the split count, so each grid gets the full (a) chain."""
    name, hidden, H, KVH, D, inter, vocab, M, bs, tile, _, form = case
    model = Model(hidden, H, KVH, D, inter, vocab, 1, 23, False)
    geo = geometry(mshim, model, M, MAX_SEQ, tile)
    assert geo.form == form
    ws = workspace(geo)
    st = Step(model, [MAX_SEQ - 1, 0, 77, 300][:M], bs, MAX_SEQ, 23, rope_table(MAX_SEQ + 1, D))
    first = None
    for kind in ("all", 33, 7, 4, 1):
        n = grid_of(kind, n_sm)
        if n < M:
            continue
        what = f"{name} n_ctas={n}"
        o = run_mega(mshim, model, st, outputs(model, st), ws, n, MAX_SEQ, tile)
        oz = run_mega(mshim, model, st, outputs(model, st), ws, n, MAX_SEQ, tile, zero_down=True)
        check_chain(mshim, n_sm, model, st, o, oz, what)
        if first is None:
            first = o
        else:
            assert_same_bits(o.q, first.q, f"{what}: q vs the full grid")
            for (k, v), (k0, v0) in zip(o.caches, first.caches):
                assert_same_bits(k, k0, f"{what}: K cache vs the full grid")
                assert_same_bits(v, v0, f"{what}: V cache vs the full grid")


@pytest.mark.parametrize("L,case", [(2, SMALL[0]), (3, SMALL[14]), (2, SMALL[1])], ids=["L2-per-warp", "L3-cta-tile", "L2-coop"])
def test_mega_layers_chain(mshim, n_sm, L, case):
    """(c): one L-layer launch against L single-layer launches, each fed the previous one's h through the embedding row of
    its token: every layer's K/V append, the final h, the last layer's q / attn / act, logits and tokens bit-identical."""
    name, hidden, H, KVH, D, inter, vocab, M, bs, tile, grid, form = case
    model = Model(hidden, H, KVH, D, inter, vocab, L, 31 + L, False)
    geo = geometry(mshim, model, M, MAX_SEQ, tile)
    assert geo.form == form
    ws = workspace(geo)
    n = grid_of(grid, n_sm)
    st = Step(model, [MAX_SEQ - 1, 5, 200, 64][:M], bs, MAX_SEQ, 31, rope_table(MAX_SEQ + 1, D))
    full = run_mega(mshim, model, st, outputs(model, st), ws, n, MAX_SEQ, tile)
    embed = model.embed
    for l in range(L):
        o = outputs(model, st)
        o.caches = [o.caches[l]]
        o = run_mega(mshim, model, st, o, ws, n, MAX_SEQ, tile, layers=[model.layers[l]], embed=embed)
        for c in range(2):
            assert_same_bits(full.caches[l][c], o.caches[0][c], f"L={L} layer {l}: KV cache")
        embed = model.embed.clone()
        embed[st.tok.long().to(DEV)] = o.h[:M]
    for name in ("h", "q", "attn", "act", "logits", "row_tok", "row_pos", "hist", "step", "fwd"):
        assert_same_bits(getattr(full, name), getattr(o, name), f"L={L}: {name}")


def test_mega_greedy_tie(mshim, n_sm):
    """Two identical lm_head rows in different passes (pairs 2 and 15998 of 16000), in different warps of the pick,
    scaled to hold the maximum logit: the lower index must win."""
    model = Model(1032, 8, 8, 128, 688, 32000, 1, 41, False)
    geo = geometry(mshim, model, 1, MAX_SEQ, 1)
    ws = workspace(geo)
    st = Step(model, [100], 16, MAX_SEQ, 41, rope_table(MAX_SEQ + 1, 128))
    lo, hi = 5, 31997
    row = model.lm_head[7].clone()
    model.lm_head[lo] = row
    model.lm_head[hi] = row
    o = run_mega(mshim, model, st, outputs(model, st), ws, n_sm, MAX_SEQ, 1)
    lg = o.logits[0].cpu()
    assert lg[lo] == lg[hi]
    sign = 1.0 if float(lg[lo]) > 0 else -1.0
    others = float(lg.abs().max())
    k = int(np.ceil(np.log2(2 * others / abs(float(lg[lo]))))) if lg[lo] != 0 else 0
    model.lm_head[lo] = (row.float() * sign * 2.0 ** max(k, 1)).to(torch.bfloat16)  # power-of-two scale: exact
    model.lm_head[hi] = model.lm_head[lo]
    o = run_mega(mshim, model, st, outputs(model, st), ws, n_sm, MAX_SEQ, 1)
    lg = o.logits[0].cpu()
    assert lg[lo] == lg[hi] and float(lg[lo]) == float(lg.max()) and int((lg == lg.max()).sum()) == 2
    assert int(o.row_tok[0]) == lo and int(o.hist[3]) == lo
    check_head(mshim, n_sm, model, st, o, "greedy tie")
