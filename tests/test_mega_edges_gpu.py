"""GPU suite (-m gpu): edges of the persistent decode kernel (csrc/mega.cu decode_mega_kernel) that the model-shaped tests
do not reach.

- Ragged LM-head passes.  The kernel hands out a matrix of P row pairs in passes of MG_CW = 8 pairs, claimed at run
  time, and the last T = 2 x MG_TAIL_PAIRS x n_ctas pairs in passes of MG_TAIL_PAIRS = 4 (claim_range); the grid is one
  CTA per SM.  Every projection of a Llama layer has P a multiple of 8, and the usual vocabularies give a tail of exactly
  T pairs, so only a vocabulary chosen from the SM count reaches a clipped last pass.
- KV block sizes 8 / 32 / 64 on the CTA-level attention forms, which stage 32-token tiles across KV blocks.
- State the kernel must leave behind: its barrier words, pass-claim counters and attention merge counters are zero
  again at exit, whatever ran in between.

Every run asserts the launch-count witness (tests/util.py::generate_counted) and is checked against the fp32 / bf16
oracles teacher-forced with the engine's own ids (tests/util.py::check_against_oracle).
"""
import os

import numpy as np
import pytest
import torch

from oracle import llama_ref, synth
from test_parity_gpu import _diag  # the diagnostics log of the parity suite
from util import assert_decode_path, check_against_oracle, generate_counted

pytestmark = pytest.mark.gpu
MG_TAIL_PAIRS = 4  # mega.cu: MG_CW / 2 row pairs per tail pass


def _prompts(vocab, lens, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, vocab, (n,), generator=g).tolist() for n in lens]


def _check(what, cfg, sd, prompts, toks, lg):
    return check_against_oracle(what, lambda: llama_ref.LlamaRef(cfg, sd, torch.float32),
                                lambda: llama_ref.LlamaRef(cfg, sd, torch.bfloat16), prompts, toks, lg, diag=_diag)


@pytest.fixture(scope="module")
def n_sm(tmp_path_factory):
    """SMs of the device = CTAs of the persistent grid (Engine::forward_mega launches one per SM)."""
    from substratus_b200 import Engine

    d = tmp_path_factory.mktemp("nsm")
    llama_ref.write_hf_dir(str(d), synth.TINY_MHA, {})
    os.remove(d / "model.safetensors")
    with Engine(str(d), {"weights": "synthetic", "max_batch": 1, "max_seq_len": 32}) as e:
        return e.info.n_sm


@pytest.mark.parametrize("pairs", ["T-1", "T", "T+7", "T+9", "16001"])
def test_lm_head_ragged_passes(tmp_path, n_sm, pairs):
    """LM head of P = V / 2 row pairs around the tail size T: T - 1 (all tail, the last pass clipped to 3 pairs), T (all
    tail, exact), T + 7 (all tail, last pass 3 pairs), T + 9 (one full pass, then a tail whose last pass holds one pair)
    and 16001 (V = 32002: many full passes, ragged tail).  Batch 1 and a ragged batch of 3 on the persistent kernel
    ("mega_max_batch": 4: the batch-4 instantiation with a padded row) and on the multi-kernel GEMV path, which has its
    own handling of a ragged last row block."""
    from substratus_b200 import Engine

    T = 2 * MG_TAIL_PAIRS * n_sm
    P = {"T-1": T - 1, "T": T, "T+7": T + 7, "T+9": T + 9, "16001": 16001}[pairs]
    cfg = dict(synth.TINY_GQA, vocab_size=2 * P)
    sd = synth.llama_state_dict(cfg, 43)
    llama_ref.write_hf_dir(str(tmp_path), cfg, sd)
    b1 = _prompts(cfg["vocab_size"], (23,), 7)
    b3 = _prompts(cfg["vocab_size"], (5, 31, 18), 8)
    for tag, mode, mega in (("persistent kernel", {"mega_max_batch": 4}, True),
                            ("multi-kernel gemv", {"use_mega": 0, "gemm_path": "gemv"}, False)):
        with Engine(str(tmp_path), dict(mode, max_batch=4, max_seq_len=64)) as e:
            for prompts in (b1, b3):
                what = f"lm_head n_sm={n_sm} T={T} P={P} ({pairs}) V={2 * P} b{len(prompts)} {tag}"
                toks, lg, launches = generate_counted(e, prompts, 5, want_logits=True)
                assert_decode_path(launches, 4, mega, what)
                assert np.isfinite(lg).all(), what
                _check(what, cfg, sd, prompts, toks, lg)


ATTN_CONFIGS = {  # the configs of test_parity_gpu.py's cooperative (G = 2) and CTA-tile (G = 8, D = 128) attention tests
    "cooperative_g2": dict(synth.TINY_GQA, hidden_size=1024, num_attention_heads=8, num_key_value_heads=4, intermediate_size=8192,
                           num_hidden_layers=2, vocab_size=1000, max_position_embeddings=1024),
    "cta_tile_g8_d128": dict(synth.TINY_GQA, hidden_size=2048, num_attention_heads=16, num_key_value_heads=2, intermediate_size=8192,
                             num_hidden_layers=2, vocab_size=1000, max_position_embeddings=1024),
}


@pytest.mark.parametrize("name", sorted(ATTN_CONFIGS))
def test_kv_block_sizes_cta_attention(tmp_path, name):
    """KV blocks of 8, 32 and 64 tokens (and 16, the reference) under the persistent kernel's CTA-level attention, in one
    ragged batch of 3: a 1-token prompt (one context split), 77 tokens, and 637 tokens whose last decode step fills
    max_seq_len = 640, i.e. ends in the final KV block whatever the block size.  Against the oracle and, bit for bit,
    against the same engine with 16-token blocks."""
    from substratus_b200 import Engine

    cfg = ATTN_CONFIGS[name]
    sd = synth.llama_state_dict(cfg, 47)
    llama_ref.write_hf_dir(str(tmp_path), cfg, sd)
    prompts = _prompts(cfg["vocab_size"], (1, 77, 637), 9)
    res = {}
    for bs in (16, 8, 32, 64):
        with Engine(str(tmp_path), {"max_batch": 4, "max_seq_len": 640, "kv_block_size": bs, "mega_max_batch": 4}) as e:
            assert e.info.kv_block_size == bs
            toks, lg, launches = generate_counted(e, prompts, 4, want_logits=True)
        what = f"{name} kv_block_size {bs} ctx {[len(p) for p in prompts]} + 3 steps"
        assert_decode_path(launches, 3, True, what)
        res[bs] = (toks, lg)
        _check(what, cfg, sd, prompts, toks, lg)
    # the persistent kernel cuts the context into splits by length alone, and the prefill does not depend on the block
    # size either: the block table is the only difference, so the results are bit-identical
    for bs in (8, 32, 64):
        err = float(np.abs(res[bs][1] - res[16][1]).max() / np.abs(res[16][1]).max())
        _diag(f"[{name} kv_block_size {bs} vs 16] logits rel err {err:.3e}; ids equal: {np.array_equal(res[bs][0], res[16][0])}")
        assert np.array_equal(res[bs][0], res[16][0]) and np.array_equal(res[bs][1], res[16][1]), (name, bs, err)


def test_state_left_between_launches(tmp_path):
    """One engine runs a batch-1 decode (persistent kernel), a batch-2 decode (graph path), a prefill, the batch-1 decode
    again on a fresh sequence with the same prompt, and the batch-2 sequences once more.  The two batch-1 runs and the
    same run on a fresh engine must give bit-identical ids and logits: the kernel leaves its grid-barrier words, pass-claim
    counters and attention merge counters at zero (the cooperative attention form runs here).  The launch counts must
    name the right path throughout, including a graph replayed after a persistent-kernel step."""
    from substratus_b200 import Engine

    cfg = ATTN_CONFIGS["cooperative_g2"]
    sd = synth.llama_state_dict(cfg, 53)
    llama_ref.write_hf_dir(str(tmp_path), cfg, sd)
    p, q, r = _prompts(cfg["vocab_size"], (40, 25, 60), 10)
    params = {"max_batch": 4, "max_seq_len": 256}
    with Engine(str(tmp_path), params) as e:
        t1, l1, n1 = generate_counted(e, [p], 6, want_logits=True)
        assert_decode_path(n1, 5, True, "first batch-1 decode")
        s2, s3 = e.seq_create(), e.seq_create()
        nxt, _ = e.prefill([s2, s3], [q, r])
        e.timing_reset()
        out, _ = e.decode([s2, s3], nxt, 3)
        assert_decode_path(e.timing().kernel_launches, 3, False, "batch-2 decode")
        t2, l2, n2 = generate_counted(e, [p], 6, want_logits=True)
        assert_decode_path(n2, 5, True, "second batch-1 decode")
        e.timing_reset()
        e.decode([s2, s3], out[:, -1], 2)  # the batch-2 graph again, right after a persistent-kernel step
        assert_decode_path(e.timing().kernel_launches, 2, False, "batch-2 decode after the persistent kernel")
    with Engine(str(tmp_path), params) as e:
        t3, l3, n3 = generate_counted(e, [p], 6, want_logits=True)
        assert_decode_path(n3, 5, True, "fresh engine")
    _diag(f"[state between launches] ids {t1.tolist()} | second run bit-identical: {np.array_equal(l2, l1)} | "
          f"fresh engine bit-identical: {np.array_equal(l3, l1)}")
    assert np.array_equal(t2, t1) and np.array_equal(l2, l1)
    assert np.array_equal(t3, t1) and np.array_equal(l3, l1)
    _check("state between launches b1", cfg, sd, [p], t1, l1)
