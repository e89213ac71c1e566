"""ctypes binding of include/ssb.h — the Python mirror of the serve host's view of the engine.

The shared library is the product; this module only marshals host buffers across the
C ABI (plain pointers and sizes).  There is no CPU fallback: if the in-tree
``substratus_b200/lib/libsubstratus_b200.so`` is missing, importing :func:`load_library`
raises, and every compute call fails with ``SSB_ENODEV`` on a box without an sm_90 GPU.

Reference seam: the generate path of the external serving image the reference's
ServerReconciler launches (internal/controller/server_controller.go:114-205;
docs/container-contract.md:50-55; the only request shape the reference ever sends is
``POST /v1/completions {"prompt", "max_tokens"}``, test/system.sh:73-78).
"""
from __future__ import annotations

import ctypes as C
import json
import os
from typing import Sequence

import numpy as np

_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib", "libsubstratus_b200.so")
_lib = None


class SsbError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"ssb error {code}: {msg}")
        self.code = code


class SsbInfo(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "vocab_size", "hidden_size", "n_layers", "n_heads", "n_kv_heads", "head_dim", "intermediate_size",
        "max_seq_len", "max_batch", "kv_block_size", "tp_size", "tp_rank", "n_sm", "device")] + [
        ("weight_bytes_per_step", C.c_int64), ("kv_bytes_per_token", C.c_int64), ("hbm_bytes_allocated", C.c_int64),
        ("model_type", C.c_char * 32), ("dtype", C.c_char * 8)]


class SsbTiming(C.Structure):
    _fields_ = [("prefill_ms", C.c_double), ("decode_ms", C.c_double), ("kernel_launches", C.c_int64),
                ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64)]


EXPORTS = [
    "ssb_engine_create", "ssb_engine_destroy", "ssb_engine_info", "ssb_seq_create", "ssb_seq_free", "ssb_seq_len",
    "ssb_kv_blocks",
    "ssb_prefill", "ssb_decode", "ssb_last_timing", "ssb_timing_reset", "ssb_tp_handle_size", "ssb_tp_export",
    "ssb_tp_connect", "ssb_bench_kernel", "ssb_debug_profile", "ssb_debug_read", "ssb_debug_dequant", "ssb_synth_fill_host", "ssb_last_error", "ssb_version", "ssb_tok_load", "ssb_tok_free", "ssb_tok_encode",
    "ssb_tok_decode", "ssb_model_read_tensor",
]


def load_library(path: str | None = None):
    """dlopen the in-tree engine library and declare the C signatures.  Raises if it is not built."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or _LIB_PATH
    if not os.path.exists(p):
        raise FileNotFoundError(
            f"{p} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU fallback for the serving path)")
    lib = C.CDLL(p)
    vp, ip, i32p, fp = C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int32), C.POINTER(C.c_float)
    lib.ssb_engine_create.argtypes = [C.c_char_p, C.c_char_p, C.POINTER(vp)]
    lib.ssb_engine_destroy.argtypes = [vp]
    lib.ssb_engine_destroy.restype = None
    lib.ssb_engine_info.argtypes = [vp, C.POINTER(SsbInfo)]
    lib.ssb_seq_create.argtypes = [vp, ip]
    lib.ssb_seq_free.argtypes = [vp, C.c_int]
    lib.ssb_seq_len.argtypes = [vp, C.c_int, ip]
    lib.ssb_kv_blocks.argtypes = [vp, ip, ip]
    lib.ssb_prefill.argtypes = [vp, ip, i32p, ip, C.c_int, i32p, fp]
    lib.ssb_decode.argtypes = [vp, ip, i32p, C.c_int, C.c_int, i32p, fp]
    lib.ssb_last_timing.argtypes = [vp, C.POINTER(SsbTiming)]
    lib.ssb_timing_reset.argtypes = [vp]
    lib.ssb_tp_handle_size.argtypes = []
    lib.ssb_tp_export.argtypes = [vp, vp]
    lib.ssb_tp_connect.argtypes = [vp, vp, C.c_int]
    lib.ssb_bench_kernel.argtypes = [vp, C.c_char_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_double),
                                     C.POINTER(C.c_int64)]
    lib.ssb_debug_profile.argtypes = [vp]
    lib.ssb_debug_profile.restype = C.c_char_p
    lib.ssb_debug_read.argtypes = [vp, C.c_char_p, fp, C.c_int64, ip, ip]
    lib.ssb_debug_dequant.argtypes = [C.c_int, vp, C.c_int64, C.c_int64, C.POINTER(C.c_uint16)]
    lib.ssb_synth_fill_host.argtypes = [C.c_uint64, C.c_uint32, C.c_int64, C.c_int64, C.c_float, C.c_float,
                                        C.POINTER(C.c_uint16)]
    lib.ssb_tok_load.argtypes = [C.c_char_p, C.POINTER(vp)]
    lib.ssb_tok_free.argtypes = [vp]
    lib.ssb_tok_free.restype = None
    lib.ssb_tok_encode.argtypes = [vp, C.c_char_p, C.c_int, i32p, C.c_int, ip]
    lib.ssb_tok_decode.argtypes = [vp, i32p, C.c_int, C.c_int, C.c_char_p, C.c_int, ip]
    lib.ssb_model_read_tensor.argtypes = [C.c_char_p, C.c_char_p, vp, C.c_int64, C.POINTER(C.c_int64), ip, C.POINTER(C.c_int64), ip]
    lib.ssb_last_error.restype = C.c_char_p
    lib.ssb_version.restype = C.c_char_p
    if path is None:
        _lib = lib
    return lib


def _check(lib, rc: int):
    if rc != 0:
        raise SsbError(rc, (lib.ssb_last_error() or b"").decode("utf-8", "replace"))


def _i32(a) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(a, dtype=np.int32))


class Engine:
    """One engine = one GPU rank holding a model (weights + paged KV cache)."""

    def __init__(self, model_dir: str, params: dict | None = None, lib_path: str | None = None):
        self._lib = load_library(lib_path)
        self._h = C.c_void_p()
        pj = json.dumps(params or {}).encode()
        _check(self._lib, self._lib.ssb_engine_create(model_dir.encode(), pj, C.byref(self._h)))
        self.info = self._info()

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self._lib.ssb_engine_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _info(self) -> SsbInfo:
        inf = SsbInfo()
        _check(self._lib, self._lib.ssb_engine_info(self._h, C.byref(inf)))
        return inf

    # ---- sequences
    def seq_create(self) -> int:
        s = C.c_int()
        _check(self._lib, self._lib.ssb_seq_create(self._h, C.byref(s)))
        return s.value

    def seq_free(self, sid: int):
        _check(self._lib, self._lib.ssb_seq_free(self._h, sid))

    def seq_len(self, sid: int) -> int:
        n = C.c_int()
        _check(self._lib, self._lib.ssb_seq_len(self._h, sid, C.byref(n)))
        return n.value

    def kv_blocks(self) -> tuple[int, int]:
        """(total, free) blocks of the KV pool; a block holds info.kv_block_size tokens."""
        t, f = C.c_int(), C.c_int()
        _check(self._lib, self._lib.ssb_kv_blocks(self._h, C.byref(t), C.byref(f)))
        return t.value, f.value

    # ---- compute
    def prefill(self, seq_ids: Sequence[int], prompts: Sequence[Sequence[int]], want_logits: bool = False):
        """Returns (next_tok [nseq] int32, logits [nseq, V] float32 or None)."""
        sid = _i32(seq_ids)
        lens = _i32([len(p) for p in prompts])
        toks = _i32(np.concatenate([np.asarray(p, dtype=np.int32) for p in prompts]))
        nxt = np.zeros(len(sid), dtype=np.int32)
        lg = np.zeros((len(sid), self.info.vocab_size), dtype=np.float32) if want_logits else None
        _check(self._lib, self._lib.ssb_prefill(
            self._h, sid.ctypes.data_as(C.POINTER(C.c_int)), toks.ctypes.data_as(C.POINTER(C.c_int32)),
            lens.ctypes.data_as(C.POINTER(C.c_int)), len(sid), nxt.ctypes.data_as(C.POINTER(C.c_int32)),
            lg.ctypes.data_as(C.POINTER(C.c_float)) if want_logits else None))
        return nxt, lg

    def decode(self, seq_ids: Sequence[int], last_tok: Sequence[int], nsteps: int, want_logits: bool = False):
        """Returns (tokens [nseq, nsteps] int32, logits [nsteps, nseq, V] float32 or None)."""
        sid = _i32(seq_ids)
        lt = _i32(last_tok)
        out = np.zeros((len(sid), nsteps), dtype=np.int32)
        lg = np.zeros((nsteps, len(sid), self.info.vocab_size), dtype=np.float32) if want_logits else None
        _check(self._lib, self._lib.ssb_decode(
            self._h, sid.ctypes.data_as(C.POINTER(C.c_int)), lt.ctypes.data_as(C.POINTER(C.c_int32)), len(sid), nsteps,
            out.ctypes.data_as(C.POINTER(C.c_int32)), lg.ctypes.data_as(C.POINTER(C.c_float)) if want_logits else None))
        return out, lg

    def generate(self, prompts: Sequence[Sequence[int]], max_new_tokens: int, want_logits: bool = False):
        """Greedy generation (HF ``generate(do_sample=False)`` semantics, no EOS stop).

        Returns (tokens [nseq, max_new_tokens], logits [max_new_tokens, nseq, V] or None)."""
        sids = [self.seq_create() for _ in prompts]
        try:
            first, lg0 = self.prefill(sids, prompts, want_logits)
            if max_new_tokens == 1:
                return first[:, None], (lg0[None] if want_logits else None)
            rest, lg = self.decode(sids, first, max_new_tokens - 1, want_logits)
            toks = np.concatenate([first[:, None], rest], axis=1)
            return toks, (np.concatenate([lg0[None], lg], axis=0) if want_logits else None)
        finally:
            for s in sids:
                self.seq_free(s)

    def timing(self) -> SsbTiming:
        t = SsbTiming()
        _check(self._lib, self._lib.ssb_last_timing(self._h, C.byref(t)))
        return t

    def timing_reset(self):
        _check(self._lib, self._lib.ssb_timing_reset(self._h))

    # ---- tensor parallel bootstrap
    def tp_export(self) -> bytes:
        n = self._lib.ssb_tp_handle_size()
        buf = C.create_string_buffer(n)
        _check(self._lib, self._lib.ssb_tp_export(self._h, C.cast(buf, C.c_void_p)))
        return buf.raw

    def tp_connect(self, all_handles: bytes):
        n = self._lib.ssb_tp_handle_size()
        assert len(all_handles) % n == 0
        buf = C.create_string_buffer(all_handles, len(all_handles))
        _check(self._lib, self._lib.ssb_tp_connect(self._h, C.cast(buf, C.c_void_p), len(all_handles) // n))

    def bench_kernel(self, which: str, rows: int = 1, ctx: int = 576, iters: int = 64):
        """(avg device ms per launch, algorithmic bytes per launch) of one kernel class of the decode step."""
        ms, by = C.c_double(), C.c_int64()
        _check(self._lib, self._lib.ssb_bench_kernel(self._h, which.encode(), rows, ctx, iters, C.byref(ms), C.byref(by)))
        return ms.value, by.value

    def profile(self) -> dict:
        """Per-kernel-class device ms since the last call (engines created with profile_forward=1)."""
        return json.loads(self._lib.ssb_debug_profile(self._h).decode())

    def debug_read(self, name: str) -> np.ndarray:
        r, c = C.c_int(), C.c_int()
        buf = np.zeros(16 * 1024 * 1024, dtype=np.float32)
        _check(self._lib, self._lib.ssb_debug_read(self._h, name.encode(), buf.ctypes.data_as(C.POINTER(C.c_float)),
                                                    buf.size, C.byref(r), C.byref(c)))
        return buf[: r.value * c.value].reshape(r.value, c.value).copy()


def synth_fill_host(seed: int, tid: int, start: int, n: int, amp: float, base: float = 0.0) -> np.ndarray:
    """bf16 bit patterns of the engine's synthetic generator (host twin; for the oracle cross-check)."""
    lib = load_library()
    out = np.zeros(n, dtype=np.uint16)
    rc = lib.ssb_synth_fill_host(seed, tid, start, n, amp, base, out.ctypes.data_as(C.POINTER(C.c_uint16)))
    _check(lib, rc)
    return out


def debug_dequant(ggml_type: int, blocks: np.ndarray, n_elems: int) -> np.ndarray:
    """Run the load-time GGUF dequant kernel on raw block bytes; returns bf16 bit patterns (tests only)."""
    lib = load_library()
    raw = np.ascontiguousarray(blocks).view(np.uint8).ravel()
    out = np.zeros(n_elems, dtype=np.uint16)
    _check(lib, lib.ssb_debug_dequant(ggml_type, raw.ctypes.data_as(C.c_void_p), raw.size, n_elems,
                                      out.ctypes.data_as(C.POINTER(C.c_uint16))))
    return out


_DTYPE_NAMES = {0: "bf16", 1: "f16", 2: "f32", 10: "q4_0", 11: "q4_k", 12: "q6_k", 13: "q8_0", 99: "other"}


def model_tensor_count(model_dir: str) -> int:
    """Number of tensors the engine's container readers find under model_dir (no device needed)."""
    lib = load_library()
    n = C.c_int64()
    _check(lib, lib.ssb_model_read_tensor(str(model_dir).encode(), None, None, 0, C.byref(n), None, None, None))
    return n.value


def model_read_tensor(model_dir: str, name: str):
    """One tensor of a Model artifact as the engine's readers see it: (dtype name, shape tuple, raw stored bytes as
    np.uint8).  Host only — safetensors / pytorch_model*.bin / GGUF (include/ssb.h: ssb_model_read_tensor)."""
    lib = load_library()
    nbytes, dt, nd = C.c_int64(), C.c_int(), C.c_int()
    shape = (C.c_int64 * 4)()
    d = str(model_dir).encode()
    _check(lib, lib.ssb_model_read_tensor(d, name.encode(), None, 0, C.byref(nbytes), C.byref(dt), shape, C.byref(nd)))
    buf = np.empty(nbytes.value, dtype=np.uint8)
    _check(lib, lib.ssb_model_read_tensor(d, name.encode(), buf.ctypes.data_as(C.c_void_p), buf.size, C.byref(nbytes), None, None, None))
    return _DTYPE_NAMES.get(dt.value, "other"), tuple(shape[i] for i in range(min(nd.value, 4))), buf


class NativeTokenizer:
    """ctypes view of the serve host's native `tokenizer.json` reader (CPU only)."""

    def __init__(self, path: str):
        self._lib = load_library()
        self._h = C.c_void_p()
        _check(self._lib, self._lib.ssb_tok_load(path.encode(), C.byref(self._h)))

    def __del__(self):
        if getattr(self, "_h", None) and self._h.value:
            self._lib.ssb_tok_free(self._h)
            self._h = C.c_void_p()

    def encode(self, text: str, add_special: bool = True):
        raw = text.encode("utf-8")
        cap = 4 * len(raw) + 16
        ids = np.zeros(cap, dtype=np.int32)
        n = C.c_int()
        _check(self._lib, self._lib.ssb_tok_encode(self._h, raw, int(add_special), ids.ctypes.data_as(C.POINTER(C.c_int32)), cap, C.byref(n)))
        return ids[: n.value].tolist()

    def decode(self, ids, skip_special: bool = True) -> str:
        a = _i32(ids)
        cap = 16 * len(a) + 64
        buf = C.create_string_buffer(cap)
        n = C.c_int()
        _check(self._lib, self._lib.ssb_tok_decode(self._h, a.ctypes.data_as(C.POINTER(C.c_int32)), len(a), int(skip_special), buf, cap, C.byref(n)))
        return buf.raw[: n.value].decode("utf-8", "replace")
