"""Kernel-level tests of the tensor-parallel exchange on ONE GPU: every allreduce kernel (kernels.cu tp_allreduce_resid /
tp_allreduce_ll / tp_reduce_push and the EPI_F32_PUSH GEMV epilogue, tp_twoshot.cu tp_allreduce2) and the persistent decode
kernel's TP modes 1 / 2 / 3 (mega.cu), launched through tests/kernel_shim.cpp as one rank with its peers staged in memory.

The exchange kernels touch their peers only through memory (peer partial buffers, flags, LL slots, gather buffers, arrival
counters and the device arrays of pointers to them), so here the "peer" buffers are ordinary device buffers.  A test writes
what the peers would already have written, launches ONE rank's kernel and checks
  1. the output h / out against a float32 emulation of the kernel's rounding, bit for bit:
         s = 0; for r in 0..size-1: s += p_r  (rank order);  out = bf16(bf16(s) + resid)  (round to nearest even twice);
  2. what it wrote into peer memory (flags = epoch; LL words {v0 bits, epoch, v1 bits, epoch} at [parity][own rank][row][pair]
     of every rank; the own gather slice; push slots and arrival counters), and that everything else in those buffers --
     filled with decoys -- is unchanged;
  3. the state it must leave clean (the two-shot `done` counter, grid_bar and the attention counters).

Sensitivity.  The staged partials cancel: each is 2^12-scale noise minus the mean over the ranks plus a 2^-2-scale remainder,
so the running fp32 sum passes through values near 2^12 while the result is small, and its bits depend on the summation
order.  Each check is paired with negative controls that the same bit comparison must reject: the reference summed in
reversed rank order and starting at the own rank (size >= 3; with two ranks fp32 addition commutes), read from the other
parity, without the residual, with the own partial counted twice.  The other parity buffer, the other LL parity (carrying
the CURRENT epoch, so that a wrong-parity read finishes with wrong bits instead of spinning) and rows >= M hold decoys.

Launch discipline.  A kernel whose wait is never met spins until its SpinGuard traps, so before every launch the host checks
that every wait the kernel will make is already met (epochs by the kernel's own formula, flags and counters at or past it,
LL words carrying it); only waits on the kernel's own writes are left unguarded.  One rank runs at a time, every launch is
synchronised, and negative controls live on the reference side only.  What this does NOT cover is memory ordering between
ranks running at the same time: that stays with test_tp_gpu.py (two or more GPUs), tools/tp_protocol_check.py and
bench.py --gpus N.
"""
import collections
import ctypes as C
import zlib

import pytest
import torch

from test_kernels_gpu import (DEV, EPI_F32, EPI_QKV_ROPE, EPI_SWIGLU, NORM_NONE, NORM_RMS, ShimProj, _struct, assert_same_bits,
                              bf, dyadic, matmul64, rope_table, run_gemv, same_bits, shim)  # noqa: F401  (shim: the fixture)
from test_mega_kernel_gpu import (MAX_SEQ, SMALL, Model, ShimMega, Step, check_head, geometry, grid_of, i32, layer_table,
                                  mega_struct, mshim, nan_rows, outputs, workspace)  # noqa: F401  (mshim: the fixture)

pytestmark = pytest.mark.gpu

INVALID_VALUE = 1          # cudaErrorInvalidValue
TP_MAX = 8                 # kernels.cu / tp_twoshot.cu / mega.cu
N_PER_STEP = 64            # allreduces per forward of a 32-layer model
WRAP_STEP = 2 ** 26 - 1    # WRAP_STEP * 64 = 2^32 - 64: allreduce 62 has epoch 2^32 - 1, allreduce 63 wraps to 0
FLAG_SENT = 0x5A5A5A5A     # flag words nobody waits on (far "ahead" of every epoch used here: a wrong index does not spin)
LL_SENT = 0x5A5A5A5A       # epoch halves of LL words that are not staged
# (tp_step, seq_in_step): step 0 / 7 / an epoch that crosses 2^32, even and odd sequence numbers (parity 0 and 1)
EPOCHS = [(0, 0), (7, 5), (WRAP_STEP, 62), (WRAP_STEP, 63)]


class ShimTpArgs(C.Structure):
    _fields_ = ([(n, C.c_void_p) for n in ("peer_partials", "peer_flags", "tp_step", "resid", "out")]
                + [(n, C.c_int) for n in ("rank", "size", "seq_in_step", "n_per_step", "parity_stride", "M", "hidden", "variant")])


class ShimTp2(C.Structure):
    _fields_ = ([(n, C.c_void_p) for n in ("peer_partials", "peer_flags", "peer_gather", "tp_step", "resid", "out", "done")]
                + [(n, C.c_int) for n in ("rank", "size", "seq_in_step", "n_per_step", "M", "hidden")]
                + [("parity_stride", C.c_longlong)])


class ShimTpPush(C.Structure):
    _fields_ = ([(n, C.c_void_p) for n in ("recv", "flags", "tp_step", "resid", "out")]
                + [(n, C.c_int) for n in ("size", "seq_in_step", "n_per_step", "M", "hidden")]
                + [(n, C.c_longlong) for n in ("arrivals_per_epoch", "parity_stride", "src_stride")])


class ShimTp(C.Structure):
    _fields_ = ([(n, C.c_void_p) for n in ("peer_partials", "peer_flags", "peer_cta_flags", "peer_ll")]
                + [(n, C.c_int) for n in ("tp_size", "tp_rank", "tp_mode")] + [("parity_stride", C.c_longlong)])


@pytest.fixture(scope="module")
def tshim(mshim):
    vp, i, ll = C.c_void_p, C.c_int, C.c_longlong
    mshim.shim_tp_allreduce_resid.argtypes = [C.POINTER(ShimTpArgs)]
    mshim.shim_tp_allreduce_ll.argtypes = [C.POINTER(ShimTpArgs), vp, ll, ll]
    mshim.shim_tp_allreduce2.argtypes = [C.POINTER(ShimTp2), i]
    mshim.shim_tp_reduce_push.argtypes = [C.POINTER(ShimTpPush)]
    mshim.shim_gemv_push.argtypes = [C.POINTER(ShimProj), vp, vp, ll, i, i, i]
    mshim.shim_gemv_grid_ctas.argtypes = [i, i, i, i]
    mshim.shim_decode_mega_tp.argtypes = [C.POINTER(ShimMega), C.POINTER(ShimTp), i]
    return mshim


@pytest.fixture(scope="module")
def n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------------------ helpers
def u32(v):
    return v & 0xFFFFFFFF


def as_i32(v):
    """a uint32 value as the int32 word the device stores"""
    v = u32(v)
    return v - 2 ** 32 if v >= 2 ** 31 else v


def epoch_of(step, seq, n_per_step):
    """the pull / LL / two-shot kernels' epoch: (uint32)step * n_per_step + seq + 1, modulo 2^32"""
    return u32(u32(step) * n_per_step + seq + 1)


def flag_met(word, epoch):
    """the kernels' wait condition (int32)(flag - epoch) >= 0 on the int32 word read back from the device"""
    return u32(int(word) - epoch) < 2 ** 31


def ptrs(ts):
    """device array of the tensors' device addresses (the kernels dereference peer-pointer arrays on the device)"""
    return torch.tensor([t.data_ptr() for t in ts], dtype=torch.int64, device=DEV)


def partials(size, shape, gen):
    """size fp32 partials (CPU) that cancel: 2^12-scale noise minus its mean over the ranks plus a 2^-2-scale remainder."""
    big = torch.randn(size, *shape, generator=gen, dtype=torch.float64) * 4096
    big -= big.mean(0, keepdim=True)
    return (big + torch.randn(size, *shape, generator=gen, dtype=torch.float64) * 0.25).float()


def with_own(size, rank, own, gen):
    """partials of the peers that cancel among themselves, with `own` (computed by the kernel under test) at `rank`"""
    peers = list(partials(size - 1, tuple(own.shape), gen))
    return torch.stack(peers[:rank] + [own.cpu().float()] + peers[rank:])


def resid_of(shape, gen):
    return (torch.randn(*shape, generator=gen) * 0.25).to(torch.bfloat16)


def decoys(shape, gen, dtype=torch.float32):
    return (torch.randn(*shape, generator=gen) * 64).to(dtype)


def reduce_ref(parts, resid):
    """float32 emulation of the exchange: s = 0; s += p_r in the given order; bf16(bf16(s) + resid) (CPU, bf16 result)"""
    s = torch.zeros_like(parts[0])
    for p in parts:
        s = s + p
    return (bf(s) + resid.float()).to(torch.bfloat16)


def check_reduce(got, parts, rank, resid, other, what, ctr, controls=True):
    """got = the rank-order reduce of parts plus resid, bit for bit; each deliberately wrong reference must be rejected.
    other: the partials of the other parity, in rank order."""
    assert_same_bits(got, reduce_ref(parts, resid), what)
    if not controls:
        return
    wrong = {"other parity": reduce_ref(other, resid), "no residual": reduce_ref(parts, torch.zeros_like(resid)),
             "own twice": reduce_ref(parts + [parts[rank]], resid)}
    if len(parts) >= 3:
        wrong["reversed"] = reduce_ref(parts[::-1], resid)
        if rank:
            wrong["from own rank"] = reduce_ref(parts[rank:] + parts[:rank], resid)
    for name, ref in wrong.items():
        assert not same_bits(got, ref), f"{what}: the reference with {name} was not rejected"
        ctr[name] += 1


def assert_controls(ctr, what, ranks):
    """every control that applies to one of the (size, rank) pairs a test ran has been rejected at least once"""
    print(f"{what}: controls rejected {dict(ctr)}")
    names = ["other parity", "no residual", "own twice"]
    names += ["reversed"] if any(size >= 3 for size, _ in ranks) else []
    names += ["from own rank"] if any(size >= 3 and rank for size, rank in ranks) else []
    for name in names:
        assert ctr[name] > 0, f"{what}: the {name} control never ran"


def ll_words(vals, epoch):
    """{v0 bits, epoch, v1 bits, epoch} per pair of vals[..., 2P] (float32, CPU) -> int32 [..., P, 4]"""
    b = vals.contiguous().view(torch.int32).reshape(*vals.shape[:-1], -1, 2)
    w = torch.empty(*b.shape[:-1], 4, dtype=torch.int32)
    w[..., 0], w[..., 2] = b[..., 0], b[..., 1]
    w[..., 1] = w[..., 3] = as_i32(epoch)
    return w


def ll_vals(words):
    """inverse of ll_words on the value halves: int32 [..., P, 4] -> float32 [..., 2P]"""
    return torch.stack([words[..., 0], words[..., 2]], -1).reshape(*words.shape[:-2], -1).view(torch.float32)


def ll_buffers(n_ranks, n_src, rows, P, gen):
    """[rank][parity][src][row][pair] uint4 receive buffers as int32 [..., 4]: decoy values, epoch halves LL_SENT"""
    ll = torch.randint(-2 ** 31, 2 ** 31 - 1, (n_ranks, 2, n_src, rows, P, 4), generator=gen, dtype=torch.int32)
    ll[..., 1] = ll[..., 3] = LL_SENT
    return ll


def run(fn, *args):
    """One launch, synchronised so that a fault is reported at the launch that caused it; returns the launcher's code."""
    torch.cuda.synchronize()
    rc = fn(*args)
    torch.cuda.synchronize()
    return rc


def bits(t):
    t = t.cpu().reshape(-1)
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16) if t.dtype == torch.bfloat16 else t


def assert_unchanged(got, want, what):
    assert bool(torch.equal(bits(got), bits(want))), what


# ------------------------------------------------------------------------------------------------------------ one-shot pull / push
class Pull:
    """Staged state of one tp_allreduce_resid / tp_allreduce_ll launch by `rank`: partial buffers [size][2 parities][rows_max
    = M + 2][hidden] (plus the push slots), flags [size][32], residual [rows_max][hidden], the live partials of this parity."""

    def __init__(self, size, rank, M, hidden, step, seq, n_per_step, gen, push=False, alias=True):
        self.size, self.rank, self.M, self.hidden, self.step, self.seq = size, rank, M, hidden, step, seq
        self.parity, self.epoch = seq & 1, epoch_of(step, seq, n_per_step)
        self.rows = M + 2
        self.ps = self.rows * hidden
        n = max(2 * self.ps, 24 * M * hidden) if push else 2 * self.ps
        self.live = partials(size, (M, hidden), gen)
        part = decoys((size, n), gen)
        for r in range(size):
            part[r, self.parity * self.ps:self.parity * self.ps + M * hidden] = self.live[r].view(-1)
        if push:  # the peers' pushes of this parity in the own buffer's slots [8 + parity * 8 + src]
            for r in range(size):
                if r != rank:
                    part[rank, self.slot(self.parity, r):self.slot(self.parity, r) + M * hidden] = self.live[r].view(-1)
        self.part = part.to(DEV)
        self.flags = torch.full((size, 32), FLAG_SENT, dtype=torch.int32, device=DEV)
        self.resid = resid_of((self.rows, hidden), gen).to(DEV)
        self.out = self.resid if alias else torch.full((self.rows, hidden), float("nan"), dtype=torch.bfloat16, device=DEV)
        self.resid0, self.out0 = self.resid.cpu(), self.out.cpu()
        self.step_t = i32([step])
        self.p_part, self.p_flags = ptrs(self.part), ptrs(self.flags)  # kept alive until the launch has finished

    def slot(self, parity, src):
        return (8 + parity * 8 + src) * self.M * self.hidden

    def other(self, part, push=False):
        """the other parity's partials in rank order (push: the slots for the peers, the partial buffer for the own rank)"""
        o, n = 1 - self.parity, self.M * self.hidden
        return [(part[self.rank, self.slot(o, r):self.slot(o, r) + n] if push and r != self.rank
                 else part[r, o * self.ps:o * self.ps + n]).view(self.M, self.hidden) for r in range(self.size)]

    def args(self, variant=0, n_per_step=N_PER_STEP):
        return _struct(ShimTpArgs, peer_partials=self.p_part, peer_flags=self.p_flags, tp_step=self.step_t,
                       resid=self.resid, out=self.out, rank=self.rank, size=self.size, seq_in_step=self.seq,
                       n_per_step=n_per_step, parity_stride=self.ps, M=self.M, hidden=self.hidden, variant=variant)

    def stage_flags(self, ahead):
        for r in range(self.size):
            if r != self.rank:
                self.flags[self.rank, r] = as_i32(self.epoch + (1 if ahead else 0))
        f = self.flags.cpu()
        assert all(flag_met(f[self.rank, r], self.epoch) for r in range(self.size) if r != self.rank), "flag precondition"
        self.flags0 = f

    def check_out(self, ctr, what, other):
        got = self.out.cpu()
        check_reduce(got[:self.M], list(self.live), self.rank, self.resid0[:self.M].float(), other, what, ctr)
        assert_same_bits(got[self.M:], self.out0[self.M:], f"{what}: out rows >= M")
        if self.out is not self.resid:
            assert_same_bits(self.resid.cpu(), self.resid0, f"{what}: resid written")

    def check_flags(self, what):
        want = self.flags0.clone()
        for r in range(self.size):
            if r != self.rank:
                want[r, self.rank] = as_i32(self.epoch)
        assert_unchanged(self.flags, want, f"{what}: flags written to the peers")


RESID_CASES = [  # (variant, size, rank, M, hidden); variant bit0 no fence, bit1 relaxed poll, bit2 push (M <= 4)
    (0, 2, 1, 1, 1032),     # one CTA, 258 float4: a partial last warp
    (1, 4, 1, 3, 5120),     # 3840 float4 on 8 CTAs
    (1, 8, 7, 300, 8192),   # 64 CTAs at the cap, 37.5 float4 per thread: a grid-stride remainder
    (2, 8, 3, 17, 5120),    # 43 CTAs, the second grid stride partial
    (3, 4, 3, 64, 1032),    # 33 CTAs
    (0, 8, 0, 4, 8192),
    (1, 2, 0, 300, 5120),
    (4, 4, 2, 1, 8192),     # push: 4 CTAs, only CTA 0 copies the own partial
    (4, 8, 5, 4, 8192),     # push: 16 CTAs
    (4, 2, 1, 3, 1032),     # push: 2 CTAs
    (6, 4, 0, 2, 5120),     # push + relaxed poll
]


@pytest.mark.parametrize("variant,size,rank,M,hidden", RESID_CASES)
def test_tp_allreduce_resid(tshim, variant, size, rank, M, hidden):
    """The one-shot pull kernel (variants 0-3) and its push variant (4, 6): output, flags, push slots; every epoch case,
    out aliasing resid (as the engine runs it) and once in a separate buffer; peers at the epoch or one allreduce ahead."""
    push = bool(variant & 4)
    ctr = collections.Counter()
    for i, (step, seq) in enumerate(EPOCHS):
        gen = torch.Generator().manual_seed(zlib.crc32(f"resid{variant}-{size}-{rank}-{M}-{hidden}-{i}".encode()))
        what = f"tp_allreduce_resid variant={variant} size={size} rank={rank} M={M} hidden={hidden} step={step} seq={seq}"
        x = Pull(size, rank, M, hidden, step, seq, N_PER_STEP, gen, push=push, alias=i != 1)
        x.stage_flags(ahead=i % 2 == 0)
        part0 = x.part.cpu()
        assert run(tshim.shim_tp_allreduce_resid, C.byref(x.args(variant))) == 0
        x.check_out(ctr, what, x.other(part0, push))
        x.check_flags(what)
        want = part0.clone()
        if push:  # the own partial lands in slot [parity][rank] of every peer; nothing else is written
            for r in range(size):
                if r != rank:
                    want[r, x.slot(x.parity, rank):x.slot(x.parity, rank) + M * hidden] = x.live[rank].view(-1)
        assert_unchanged(x.part, want, f"{what}: partial buffers / push slots")
    assert_controls(ctr, f"tp_allreduce_resid variant={variant}", [(size, rank)])


# ------------------------------------------------------------------------------------------------------------ LL
LL_CASES = [  # (size, rank, M, hidden)
    (2, 1, 1, 1032),   # 516 pairs: an odd pair count
    (4, 2, 4, 8192),   # 64 x 256 pairs exactly
    (8, 7, 4, 8196),   # 4 x 4098 pairs: the grid-stride loop goes round twice
    (8, 3, 3, 1032),
    (4, 0, 2, 8196),
    (2, 0, 4, 8192),
]


class Ll(Pull):
    """Pull plus LL receive buffers [size][2][n_src][rows][P] (int32 x 4): the peers' words of this parity staged in the
    own buffer with the epoch, the other parity's slots holding decoys that carry the current epoch too."""

    def __init__(self, size, rank, M, hidden, step, seq, gen, n_src=TP_MAX, ll_rows=4, alias=True):
        super().__init__(size, rank, M, hidden, step, seq, N_PER_STEP, gen, alias=alias)
        P = hidden // 2
        self.P, self.n_src, self.ll_rows = P, n_src, ll_rows
        ll = ll_buffers(size, n_src, ll_rows, P, gen)
        self.other_vals = decoys((size, M, hidden), gen)
        for r in range(size):  # [..., :2P]: an odd hidden (refused) leaves its last element out
            if r != rank:
                ll[rank, self.parity, r, :M] = ll_words(self.live[r][:, :2 * P], self.epoch)
            ll[rank, 1 - self.parity, r, :M] = ll_words(self.other_vals[r][:, :2 * P], self.epoch)
        w = ll[rank, self.parity]
        assert all(bool((w[r, :M, :, 1] == as_i32(self.epoch)).all() and (w[r, :M, :, 3] == as_i32(self.epoch)).all())
                   for r in range(size) if r != rank), "LL precondition"
        self.ll0 = ll
        self.ll = ll.to(DEV)
        self.p_ll = ptrs(self.ll)
        self.flags0 = self.flags.cpu()

    def launch(self, tshim):
        src = self.ll_rows * self.P
        return run(tshim.shim_tp_allreduce_ll, C.byref(self.args()), self.p_ll.data_ptr(), self.n_src * src, src)


@pytest.mark.parametrize("size,rank,M,hidden", LL_CASES)
def test_tp_allreduce_ll(tshim, size, rank, M, hidden):
    """The LL push allreduce of the multi-kernel decode: output; the own words {v0, epoch, v1, epoch} at [parity][rank][row]
    of every rank's buffer (own included); nothing else written (the peers' partial buffers are never read)."""
    ctr = collections.Counter()
    for i, (step, seq) in enumerate(EPOCHS):
        gen = torch.Generator().manual_seed(zlib.crc32(f"ll-{size}-{rank}-{M}-{hidden}-{i}".encode()))
        what = f"tp_allreduce_ll size={size} rank={rank} M={M} hidden={hidden} step={step} seq={seq}"
        x = Ll(size, rank, M, hidden, step, seq, gen, alias=i != 1)
        part0 = x.part.cpu()
        assert x.launch(tshim) == 0
        other = [x.other_vals[r] if r != rank else x.other(part0)[r] for r in range(size)]
        x.check_out(ctr, what, other)
        want = x.ll0.clone()
        for r in range(size):
            want[r, x.parity, rank, :M] = ll_words(x.live[rank], x.epoch)
        assert_unchanged(x.ll, want, f"{what}: LL words")
        assert_unchanged(x.part, part0, f"{what}: partial buffers")
        assert_unchanged(x.flags, x.flags0, f"{what}: flags")
    assert_controls(ctr, "tp_allreduce_ll", [(size, rank)])


# ------------------------------------------------------------------------------------------------------------ two-shot
TWO_CASES = [  # (size, rank, M, hidden, n_sm cap: "all" = the device)
    (4, 1, 3, 1032, "all"),     # 774 float4: slices of 193 / 194
    (8, 7, 3, 1032, "all"),     # 96.75 float4 per slice
    (4, 2, 1, 8, "all"),        # 2 float4 for 4 ranks: empty slices
    (8, 3, 1, 20, "all"),       # 5 float4 for 8 ranks
    (8, 5, 600, 8192, "all"),   # 153600 float4 per slice: the grid is capped at the SM count
    (8, 0, 512, 8192, 64),      # a prefill at TP 8, grid capped at 64
    (2, 1, 17, 5120, 7),
]


@pytest.mark.parametrize("size,rank,M,hidden,cap", TWO_CASES)
def test_tp_allreduce2(tshim, n_sm, size, rank, M, hidden, cap):
    """The two-shot allreduce: the own slice against the reference, the peers' slices equal to their staged gather bits,
    the own gather slice written and nothing else, flags [own] = [8 + own] = epoch at every peer, `done` back to 0."""
    ctr = collections.Counter()
    total4 = M * hidden // 4
    lo, hi = total4 * rank // size, total4 * (rank + 1) // size
    for i, (step, seq) in enumerate(EPOCHS):
        gen = torch.Generator().manual_seed(zlib.crc32(f"two-{size}-{rank}-{M}-{hidden}-{i}".encode()))
        what = f"tp_allreduce2 size={size} rank={rank} M={M} hidden={hidden} step={step} seq={seq}"
        x = Pull(size, rank, M, hidden, step, seq, N_PER_STEP, gen, alias=i != 1)
        gather = decoys((size, x.rows * hidden), gen, torch.bfloat16)
        x.gather = gather.to(DEV)
        for r in range(size):
            if r != rank:
                x.flags[rank, r] = x.flags[rank, TP_MAX + r] = as_i32(x.epoch + (1 if i % 2 == 0 else 0))
        f = x.flags.cpu()
        assert all(flag_met(f[rank, r], x.epoch) and flag_met(f[rank, TP_MAX + r], x.epoch) for r in range(size) if r != rank)
        done = torch.zeros(1, dtype=torch.int32, device=DEV)
        part0 = x.part.cpu()
        p_gather = ptrs(x.gather)
        s = _struct(ShimTp2, peer_partials=x.p_part, peer_flags=x.p_flags, peer_gather=p_gather, tp_step=x.step_t,
                    resid=x.resid, out=x.out, done=done, rank=rank, size=size, seq_in_step=seq, n_per_step=N_PER_STEP, M=M,
                    hidden=hidden, parity_stride=x.ps)
        assert run(tshim.shim_tp_allreduce2, C.byref(s), grid_of(cap, n_sm)) == 0
        got = x.out.cpu().view(-1)
        flat = lambda t: t.reshape(-1)[4 * lo:4 * hi]
        if hi > lo:  # controls where the slice is long enough for a wrong order to show
            check_reduce(flat(got), [flat(p) for p in x.live], rank, flat(x.resid0[:M].float()),
                         [flat(p) for p in x.other(part0)], what, ctr, controls=hi - lo >= 64)
        for p in range(size):
            if p != rank:
                plo, phi = total4 * p // size, total4 * (p + 1) // size
                assert_same_bits(got[4 * plo:4 * phi], gather[p, 4 * plo:4 * phi], f"{what}: slice of rank {p}")
        assert_same_bits(got[M * hidden:], x.out0.view(-1)[M * hidden:], f"{what}: out rows >= M")
        want = gather.clone()
        want[rank, 4 * lo:4 * hi] = got[4 * lo:4 * hi]
        assert_same_bits(x.gather.cpu(), want, f"{what}: gather buffers")
        want = f.clone()
        for r in range(size):
            if r != rank:
                want[r, rank] = want[r, TP_MAX + rank] = as_i32(x.epoch)
        assert_unchanged(x.flags, want, f"{what}: flags written to the peers")
        assert_unchanged(x.part, part0, f"{what}: partial buffers")
        assert int(done) == 0, f"{what}: done counter not reset"
    if hi - lo >= 64:
        assert_controls(ctr, "tp_allreduce2", [(size, rank)])


# ------------------------------------------------------------------------------------------------------------ push GEMV + reduce
PUSH_CASES = [  # (size, rank, M, N = hidden, K = this rank's q_rows or inter, tp_step)
    (8, 3, 1, 8192, 1024, 1),            # Llama-2-70B o_proj at TP 8
    (4, 2, 3, 8192, 28672, 7),           # K = 28672: the 4-row tile does not fit, 2 rows of CTAs
    (2, 1, 4, 5120, 6912, 2 ** 31 - 1),  # 13B down at TP 2; the arrival target passes 2^32
    (4, 0, 2, 248, 4096, 7),             # P = 124 pairs: fewer CTAs than SMs
    (8, 7, 4, 4096, 1376, 1),            # 7B down at TP 8
]


@pytest.mark.parametrize("size,rank,M,N,K,step", PUSH_CASES)
def test_gemv_push_and_reduce(tshim, n_sm, size, rank, M, N, K, step):
    """EPI_F32_PUSH: the float64-exact partial in slot [parity][rank] of every rank's receive buffer, rows >= M and every
    other slot untouched, each destination's arrival counter [rank] up by exactly gemv_grid_ctas.  Then the peers' slots
    and counters are staged and tp_reduce_push sums the slots in rank order onto the residual."""
    hidden, mb = N, 4  # receive buffers [2][8][max_batch = 4][hidden], as Engine sizes them
    src_stride, parity_stride = mb * hidden, 8 * mb * hidden
    arrivals = tshim.shim_gemv_grid_ctas(M, N, K, n_sm)
    ctr = collections.Counter()
    for seq in (2, 5):
        gen = torch.Generator().manual_seed(zlib.crc32(f"push-{size}-{rank}-{M}-{N}-{K}-{seq}".encode()))
        dgen = torch.Generator(device=DEV).manual_seed(seq * 1000 + N + K)
        what = f"push size={size} rank={rank} M={M} N={N} K={K} step={step} seq={seq}"
        parity = seq & 1
        target = ((u32(step - 1) * N_PER_STEP + seq + 1) * arrivals) % 2 ** 64
        W, x = dyadic((N, K), dgen), dyadic((M, K), dgen)
        exact = matmul64(x, W).float()
        recv = decoys((size, 2 * parity_stride), gen)
        recv_d = recv.to(DEV)
        cnt = torch.randint(0, 2 ** 40, (size, size), generator=gen, dtype=torch.int64)
        cnt[rank, rank] = target - arrivals
        cnt_d = cnt.to(DEV)
        off = parity * parity_stride + rank * src_stride
        s = _struct(ShimProj, W=W, x=x, N=N, K=K, ldx=K, M=M, ld_out=hidden)
        p_recv, p_cnt = ptrs(recv_d), ptrs(cnt_d)
        rc = run(tshim.shim_gemv_push, C.byref(s), p_recv.data_ptr(), p_cnt.data_ptr(), off, size, rank, n_sm)
        assert rc == 0
        want = cnt.clone()
        want[:, rank] += arrivals
        assert_unchanged(cnt_d, want, f"{what}: arrival counters (+{arrivals} each at [rank])")
        want = recv.clone()
        want[:, off:off + M * hidden] = exact.reshape(-1)
        assert_unchanged(recv_d, want, f"{what}: push slots")
        # the reduce: the peers' slots of this parity, counters at the target (or one allreduce ahead)
        live = with_own(size, rank, exact, gen)
        for r in range(size):
            if r != rank:
                o = parity * parity_stride + r * src_stride
                recv_d[rank, o:o + M * hidden] = live[r].reshape(-1).to(DEV)
                cnt_d[rank, r] = target + (arrivals if r % 2 else 0)
        c = cnt_d[rank].cpu()
        assert all(int(v) >= target for v in c), "arrival-counter precondition"
        recv1, cnt1 = recv_d.cpu(), cnt_d.cpu()
        resid = resid_of((mb, hidden), gen).to(DEV)
        resid0 = resid.cpu()
        out = resid if seq == 2 else torch.full((mb, hidden), float("nan"), dtype=torch.bfloat16, device=DEV)
        out0 = out.cpu()
        step_t = i32([step])
        t = _struct(ShimTpPush, recv=recv_d[rank], flags=cnt_d[rank], tp_step=step_t, resid=resid, out=out, size=size,
                    seq_in_step=seq, n_per_step=N_PER_STEP, M=M, hidden=hidden, arrivals_per_epoch=arrivals,
                    parity_stride=parity_stride, src_stride=src_stride)
        assert run(tshim.shim_tp_reduce_push, C.byref(t)) == 0
        other = [recv1[rank, (1 - parity) * parity_stride + r * src_stride:][:M * hidden].view(M, hidden) for r in range(size)]
        check_reduce(out.cpu()[:M], list(live), rank, resid0[:M].float(), other, what, ctr)
        assert_same_bits(out.cpu()[M:], out0[M:], f"{what}: out rows >= M")
        assert_unchanged(recv_d, recv1, f"{what}: receive buffers after the reduce")
        assert_unchanged(cnt_d, cnt1, f"{what}: counters after the reduce")
    assert_controls(ctr, "push", [(size, rank)])


# ------------------------------------------------------------------------------------------------------------ refusals
def refused_pull(tshim, kind):
    """Buffers sized and staged for the refused shape, so that a launch that slipped through would still complete."""
    gen = torch.Generator().manual_seed(zlib.crc32(kind.encode()))
    if kind == "resid size 9":
        x = Pull(9, 4, 2, 1032, 7, 0, N_PER_STEP, gen)
        x.stage_flags(False)
        return x, lambda: run(tshim.shim_tp_allreduce_resid, C.byref(x.args()))
    if kind == "resid hidden 1030":
        x = Pull(4, 1, 1, 1030, 7, 0, N_PER_STEP, gen)
        x.stage_flags(False)
        return x, lambda: run(tshim.shim_tp_allreduce_resid, C.byref(x.args()))
    if kind == "ll size 9":
        x = Ll(9, 4, 2, 1032, 7, 0, gen, n_src=9)
    elif kind == "ll M 5":
        x = Ll(4, 1, 5, 1032, 7, 0, gen, ll_rows=5)
    else:  # "ll hidden 1031": one row, so that every pair stays 8-byte aligned
        x = Ll(4, 1, 1, 1031, 7, 0, gen)
    return x, lambda: x.launch(tshim)


@pytest.mark.parametrize("kind", ["resid size 9", "resid hidden 1030", "ll size 9", "ll M 5", "ll hidden 1031"])
def test_exchange_refusals_pull(tshim, kind):
    """Shapes the one-shot and LL launchers must refuse with cudaErrorInvalidValue, writing nothing."""
    x, launch = refused_pull(tshim, kind)
    part0, flags0 = x.part.cpu(), x.flags.cpu()
    assert launch() == INVALID_VALUE
    assert_unchanged(x.out, x.out0, f"{kind}: out written")
    assert_unchanged(x.part, part0, f"{kind}: partials written")
    assert_unchanged(x.flags, flags0, f"{kind}: flags written")
    if isinstance(x, Ll):
        assert_unchanged(x.ll, x.ll0, f"{kind}: LL words written")


@pytest.mark.parametrize("size,hidden", [(9, 1032), (4, 1030)])
def test_exchange_refusals_two_shot_and_push(tshim, n_sm, size, hidden):
    """tp_allreduce2 and tp_reduce_push refuse size 9 and hidden % 4 != 0, writing nothing."""
    gen = torch.Generator().manual_seed(size * 100 + hidden)
    M, rank = 1, size - 1
    x = Pull(size, rank, M, hidden, 7, 0, N_PER_STEP, gen)
    for r in range(size):
        if r != rank:
            x.flags[rank, r] = x.flags[rank, TP_MAX + r] = as_i32(x.epoch)
    gather = decoys((size, x.rows * hidden), gen, torch.bfloat16).to(DEV)
    done = torch.zeros(1, dtype=torch.int32, device=DEV)
    part0, flags0, gather0 = x.part.cpu(), x.flags.cpu(), gather.cpu()
    p_gather = ptrs(gather)
    s = _struct(ShimTp2, peer_partials=x.p_part, peer_flags=x.p_flags, peer_gather=p_gather, tp_step=x.step_t,
                resid=x.resid, out=x.out, done=done, rank=rank, size=size, seq_in_step=0, n_per_step=N_PER_STEP, M=M,
                hidden=hidden, parity_stride=x.ps)
    assert run(tshim.shim_tp_allreduce2, C.byref(s), n_sm) == INVALID_VALUE
    # push reduce: every counter far past any target
    recv = decoys((2 * TP_MAX * 4 * hidden + size * 4 * hidden,), gen).to(DEV)
    cnt = torch.full((size,), 2 ** 62, dtype=torch.int64, device=DEV)
    recv0 = recv.cpu()
    step_t = i32([7])
    t = _struct(ShimTpPush, recv=recv, flags=cnt, tp_step=step_t, resid=x.resid, out=x.out, size=size, seq_in_step=0,
                n_per_step=N_PER_STEP, M=M, hidden=hidden, arrivals_per_epoch=132, parity_stride=max(8, size) * 4 * hidden,
                src_stride=4 * hidden)
    assert run(tshim.shim_tp_reduce_push, C.byref(t)) == INVALID_VALUE
    assert_unchanged(x.out, x.out0, "out written")
    assert_unchanged(x.part, part0, "partials written")
    assert_unchanged(x.flags, flags0, "flags written")
    assert_unchanged(gather, gather0, "gather written")
    assert_unchanged(recv, recv0, "receive buffer written")
    assert int(done) == 0


# ------------------------------------------------------------------------------------------------------------ persistent kernel
MEGA_CASES = [  # (SMALL case, grid): head_dim 128, hidden 1032 (P = 516: uneven part_range at every grid), M in 1..4
    ("d128g1-warp", 1), ("d128g2-warp", 7), ("d128g4-warp", "all"), ("d128g8-warp", "all"), ("d128g16-cta", 7),
    ("d128g2-coop", "all"),
]
CTA_FLAG_STRIDE = 256  # mega.cu MG_CTA_FLAG_STRIDE


class MegaTp:
    """Exchange state of one persistent TP launch as `rank` of `size` with ONE layer: the step makes exactly two allreduces
    (O: seq 0, parity 0, epoch e0; down: seq 1, parity 1, epoch e1 = e0 + 1), so both can be staged before the launch.
    Two layers would need a peer to rewrite a parity buffer between allreduces, which a single-rank launch cannot stage.
    partials [size][2][4 rows][hidden], flags [size][32], per-CTA flags [size][8][256], LL [size][2][8][4][P]."""

    def __init__(self, size, rank, mode, M, hidden, n_ctas, f0, live_o, live_d, gen):
        self.size, self.rank, self.mode, self.M, self.hidden = size, rank, mode, M, hidden
        base = u32((f0 + 1) * 2)  # the kernel bumps fwd_counter to f0 + 1; 2 allreduces per forward
        self.e = (u32(base + 1), u32(base + 2))
        self.ps = 4 * hidden
        part = decoys((size, 2 * self.ps), gen)
        flags = torch.full((size, 32), FLAG_SENT, dtype=torch.int32)
        cta = torch.full((size, TP_MAX * CTA_FLAG_STRIDE), FLAG_SENT, dtype=torch.int32)
        ll = ll_buffers(size, TP_MAX, 4, hidden // 2, gen)
        for r in range(size):
            if r == rank:
                continue
            for par, live in enumerate((live_o, live_d)):
                part[r, par * self.ps:par * self.ps + M * hidden] = live[r].reshape(-1)
                if mode == 3:
                    ll[rank, par, r, :M] = ll_words(live[r], self.e[par])
            if mode == 1:
                flags[rank, r] = as_i32(self.e[1])  # at or past both allreduces
            if mode == 2:
                cta[rank, r * CTA_FLAG_STRIDE:r * CTA_FLAG_STRIDE + n_ctas] = as_i32(self.e[1])
        peers = [r for r in range(size) if r != rank]
        if mode == 1:
            assert all(flag_met(flags[rank, r], e) for r in peers for e in self.e), "flag precondition"
        if mode == 2:
            assert all(flag_met(cta[rank, r * CTA_FLAG_STRIDE + c], e) for r in peers for c in range(n_ctas) for e in self.e)
        if mode == 3:
            for par in (0, 1):
                w = ll[rank, par, peers, :M]
                assert bool((w[..., 1] == as_i32(self.e[par])).all() and (w[..., 3] == as_i32(self.e[par])).all()), "LL precondition"
        self.part0, self.flags0, self.cta0, self.ll0 = part, flags, cta, ll
        self.part, self.flags, self.cta, self.ll = part.to(DEV), flags.to(DEV), cta.to(DEV), ll.to(DEV)
        self.ptrs = [ptrs(t) for t in (self.part, self.flags, self.cta, self.ll)]  # kept alive until the launch has finished

    def struct(self):
        return _struct(ShimTp, peer_partials=self.ptrs[0], peer_flags=self.ptrs[1], peer_cta_flags=self.ptrs[2],
                       peer_ll=self.ptrs[3], tp_size=self.size, tp_rank=self.rank, tp_mode=self.mode, parity_stride=self.ps)

    def own_partials(self):
        """the own O and down partials the kernel left: its partial buffer (modes 1, 2) or its LL slots in a peer's buffer"""
        M, h = self.M, self.hidden
        if self.mode == 3:
            peer = (self.rank + 1) % self.size
            return [ll_vals(self.ll[peer, par, self.rank, :M].cpu()) for par in (0, 1)]
        p = self.part.cpu()
        return [p[self.rank, par * self.ps:par * self.ps + M * h].view(M, h) for par in (0, 1)]

    def check_written(self, own, n_ctas, what):
        """flags / per-CTA flags / LL words at every peer carry the right epoch and bits; nothing else written"""
        M, h, rank = self.M, self.hidden, self.rank
        part, flags, cta, ll = self.part0.clone(), self.flags0.clone(), self.cta0.clone(), self.ll0.clone()
        for par in (0, 1):
            if self.mode == 3:
                for r in range(self.size):
                    ll[r, par, rank, :M] = ll_words(own[par], self.e[par])
            else:
                part[rank, par * self.ps:par * self.ps + M * h] = own[par].reshape(-1)
        for r in range(self.size):
            if r != rank and self.mode == 1:
                flags[r, rank] = as_i32(self.e[1])
            if r != rank and self.mode == 2:
                cta[r, rank * CTA_FLAG_STRIDE:rank * CTA_FLAG_STRIDE + n_ctas] = as_i32(self.e[1])
        assert_unchanged(self.part, part, f"{what}: partial buffers")
        assert_unchanged(self.flags, flags, f"{what}: flags")
        assert_unchanged(self.cta, cta, f"{what}: per-CTA flags")
        assert_unchanged(self.ll, ll, f"{what}: LL words")


def run_mega_tp(tshim, model, st, ws, n, tile, x, zero_down=False):
    o = outputs(model, st)
    table = layer_table(model.layers, o.caches, model.zero_down if zero_down else None)
    s = mega_struct(model, st.M, MAX_SEQ, tile, st, o, ws, table)
    assert run(tshim.shim_decode_mega_tp, C.byref(s), C.byref(x.struct()), n) == 0
    assert int(ws.bar.abs().sum()) == 0, "grid_bar words not zero after the launch"
    assert int(ws.counters.abs().sum()) == 0, "attention merge counters not zero after the launch"
    return o


def gemv_f32(shim, n_sm, W, x, N, K):
    out = torch.full((x.shape[0], N), float("nan"), device=DEV)
    run_gemv(shim, EPI_F32, NORM_NONE, n_sm, W=W, x=x.contiguous(), N=N, K=K, ldx=K, M=x.shape[0], out_f32=out, ld_out=N)
    return out.cpu()


@pytest.mark.parametrize("mode", [1, 2, 3])
@pytest.mark.parametrize("name,grid", MEGA_CASES, ids=[c[0] for c in MEGA_CASES])
def test_mega_tp(tshim, n_sm, name, grid, mode):
    """decode_mega_kernel<.., TP=true> as rank 0 and rank size-1 of 2 and 4, teacher-forced as test_mega_kernel_gpu's
    check_chain: q / K / V, the own O and down partials bit-identical to the EPI_F32 GEMV on the observed attn / act, h after
    O (seen through a launch with wdown = 0 and zero staged down partials) and after down equal to the rank-order reduce of
    (own, staged peers) plus the residual, then logits and the greedy pick; flags, per-CTA flags and LL words written to the
    peers; grid_bar and the attention counters back to zero."""
    case = next(c for c in SMALL if c[0] == name)
    _, hidden, H, KVH, D, inter, vocab, M, bs, tile, _, form = case
    seed = zlib.crc32(f"tp-{name}".encode()) % 100000
    model = Model(hidden, H, KVH, D, inter, vocab, 1, seed, False)
    geo = geometry(tshim, model, M, MAX_SEQ, tile)
    assert geo.form == form and D == 128
    n = grid_of(grid, n_sm)
    ws = workspace(geo)
    st = Step(model, [MAX_SEQ - 1, 0, 77, 300][:M], bs, MAX_SEQ, seed, rope_table(MAX_SEQ + 1, D))
    w = model.layers[0]
    h0 = model.embed[st.tok.long().to(DEV)]
    ctr = collections.Counter()
    for size in (2, 4):
        for rank in (0, size - 1):
            what = f"{name} mode={mode} size={size} rank={rank} n_ctas={n}"
            gen = torch.Generator().manual_seed(zlib.crc32(what.encode()))
            zero = torch.zeros(M, hidden)  # the own rank's entry is never staged
            live_o, live_d = with_own(size, rank, zero, gen), with_own(size, rank, zero, gen)
            x = MegaTp(size, rank, mode, M, hidden, n, 5, live_o, live_d, gen)
            o = run_mega_tp(tshim, model, st, ws, n, tile, x)
            xz = MegaTp(size, rank, mode, M, hidden, n, 5, live_o, torch.zeros_like(live_d), gen)
            oz = run_mega_tp(tshim, model, st, ws, n, tile, xz, zero_down=True)
            for t in ("h", "q", "attn", "act", "logits"):
                assert nan_rows(getattr(o, t), M) and nan_rows(getattr(oz, t), M), f"{what}: {t} rows >= M written"
            for t in ("q", "attn", "act"):
                assert_same_bits(getattr(oz, t), getattr(o, t), f"{what}: {t} with wdown = 0")
            # q and the K/V append
            q_ref = torch.full((M, model.q_rows), float("nan"), device=DEV, dtype=torch.bfloat16)
            kc, vc = st.caches[0][0].clone(), st.caches[0][1].clone()
            run_gemv(tshim, EPI_QKV_ROPE, NORM_RMS, n_sm, W=w.wqkv, x=h0, N=model.q_rows + 2 * model.kv_rows, K=hidden,
                     ldx=hidden, M=M, norm_w=w.ln1, eps=1e-5, q_out=q_ref, q_rows=model.q_rows, kv_rows=model.kv_rows,
                     head_dim=D, kcache=kc, vcache=vc, block_table=st.kv.bt_dev, bt_stride=st.kv.stride,
                     row_slot=i32(st.slot.tolist()), row_pos=i32(st.pos.tolist()), rope_cs=st.table, block_size=st.bs,
                     kvh=model.KVH)
            assert_same_bits(o.q[:M], q_ref, f"{what}: q")
            assert_same_bits(o.caches[0][0], kc, f"{what}: K cache")
            assert_same_bits(o.caches[0][1], vc, f"{what}: V cache")
            # O: the own partial, then the reduce onto the embedding rows (h with wdown = 0 and zero down partials)
            own_o, own_d = x.own_partials()
            own_oz, _ = xz.own_partials()
            want_o = gemv_f32(tshim, n_sm, w.wo, o.attn[:M], hidden, model.q_rows)
            assert_same_bits(own_o, want_o, f"{what}: own O partial")
            assert_same_bits(own_oz, want_o, f"{what}: own O partial (wdown = 0)")
            parts = [want_o if r == rank else live_o[r] for r in range(size)]
            other = [own_o if r == rank else live_d[r] for r in range(size)]
            check_reduce(oz.h[:M].cpu(), parts, rank, h0.cpu().float(), other, f"{what}: h after O", ctr)
            # gate/up + SwiGLU on the observed h_mid
            act = torch.full((M, inter), float("nan"), device=DEV, dtype=torch.bfloat16)
            run_gemv(tshim, EPI_SWIGLU, NORM_RMS, n_sm, W=w.wgu, x=oz.h[:M].contiguous(), N=2 * inter, K=hidden, ldx=hidden,
                     M=M, norm_w=w.ln2, eps=1e-5, out_bf16=act, ld_out=inter)
            assert_same_bits(o.act[:M], act, f"{what}: act")
            # down: the own partial, then the reduce onto h_mid
            want_d = gemv_f32(tshim, n_sm, w.wdown, o.act[:M], hidden, inter)
            assert_same_bits(own_d, want_d, f"{what}: own down partial")
            parts = [want_d if r == rank else live_d[r] for r in range(size)]
            other = [own_d if r == rank else live_o[r] for r in range(size)]
            check_reduce(o.h[:M].cpu(), parts, rank, oz.h[:M].cpu().float(), other, f"{what}: h after down", ctr)
            check_head(tshim, n_sm, model, st, o, what)
            x.check_written([own_o, own_d], n, what)
            xz.check_written(xz.own_partials(), n, f"{what} (wdown = 0)")
    assert_controls(ctr, f"{name} mode={mode}", [(2, 0), (2, 1), (4, 0), (4, 3)])
