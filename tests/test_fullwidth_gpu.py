"""GPU suite, TRUE MODEL WIDTHS (few layers): the CUDA path through the C ABI against the HF-pinned oracle at the widths
BASELINE.json's configs run at — K tails, 8192-wide rows, d=64 Falcon heads and GQA 64/8 at real tile counts:

    llama2-7b   h=4096  H=32  KV=32 d=128 I=11008 V=32000   (config 2)
    llama2-13b  h=5120  H=40  KV=40 d=128 I=13824 V=32000   (config 3; weights arrive as a Q4_0 GGUF `model.bin`)
    llama2-70b  h=8192  H=64  KV=8  d=128 I=28672 V=32000   (config 5)
    falcon-40b  h=8192  H=128 KV=8  d=64  ffn=32768 V=65024 (config 4)

each with 2 decoder layers (the per-layer arithmetic is what the width changes; depth is covered by
test_full_depth_7b_vs_fp32_oracle below), at batch 1 (persistent kernel / GEMV path) and batch 8 (wgmma stream-K
path), prompts of 40-70 tokens crossing 16-token KV blocks, 4 decode steps.

Oracle: oracle/llama_ref.py / falcon_ref.py (bit-pinned to HF transformers 5.5.0 eager in tests/test_oracle.py), run on
the box's host cores in fp32 (truth) and bf16 (noise yardstick) as ONE teacher-forced pass over prompt + the engine's own
greedy continuation.  Tolerance = tests/test_parity_gpu.py::_assert_parity (north_star's 1e-3 on the mean against the
fp32 truth, relative to the CPU bf16 oracle's own error).  Token check: every greedy id the engine picked must be the
fp32 oracle's argmax for the same context, unless the oracle's margin between the two candidates is below the measured
bf16 noise (a rounding-level tie).

Weights are the seeded synthetic values of oracle/synth.py: created on the device by the engine ("weights":
"synthetic"; bit-exact with the oracle's generator — test_parity_gpu.py::test_synthetic_weights_match_oracle) and on the
host through the generator's C twin (oracle.synth.set_fast_fill) so that 2.4 G parameters take seconds.
Decode attention keeps P in fp32 for P.V where HF rounds P to bf16 (DESIGN.md section 2) — the one deliberate
deviation from the oracle's rounding points; it is inside every number this file prints.
"""
import os

import numpy as np
import pytest
import torch

import util
from oracle import falcon_ref as fr
from oracle import llama_ref, synth
from util import assert_decode_path, generate_counted

pytestmark = pytest.mark.gpu
TOL = 1e-3

WIDTHS = {
    "llama2-7b": dict(synth.LLAMA2_7B, num_hidden_layers=2),
    "llama2-70b": dict(synth.LLAMA2_70B, num_hidden_layers=2),
    "falcon-40b": dict(fr.FALCON_40B, num_hidden_layers=2),
}
LENS8 = (40, 47, 53, 58, 61, 64, 66, 70)  # ragged batch; 64 = exactly 4 KV blocks, 61..64 + 4 steps cross a block edge


def _diag(msg):
    os.makedirs("gpurun_out", exist_ok=True)
    with open("gpurun_out/parity_fullwidth.txt", "a") as f:
        f.write(msg + "\n")
    print(msg)


@pytest.fixture(scope="module", autouse=True)
def _fast_synth():
    from substratus_b200.engine import synth_fill_host

    synth.set_fast_fill(synth_fill_host)
    torch.set_num_threads(max(1, min(32, len(os.sched_getaffinity(0)))))
    yield
    synth.set_fast_fill(None)


def _prompts(vocab, lens, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, vocab, (n,), generator=g).tolist() for n in lens]


def check_against_oracle(what, make32, makebf, prompts, toks, lg):
    """toks [nseq, n], lg [n, nseq, V] from the engine (criterion: tests/util.py::check_against_oracle)."""
    return util.check_against_oracle(f"fullwidth {what}", make32, makebf, prompts, toks, lg, diag=_diag, tol=TOL)


def _model_dir(tmp_path, cfg):
    llama_ref.write_hf_dir(str(tmp_path), cfg, {})
    os.remove(tmp_path / "model.safetensors")
    return str(tmp_path)


@pytest.mark.parametrize("name", sorted(WIDTHS))
def test_true_width_vs_oracle(tmp_path, name):
    from substratus_b200 import Engine

    cfg = WIDTHS[name]
    falcon = cfg["model_type"] == "falcon"
    seed = 31
    specs = fr.falcon_tensor_specs(cfg) if falcon else synth.llama_tensor_specs(cfg)
    Ref = fr.FalconRef if falcon else llama_ref.LlamaRef
    # one materialised bf16 state dict shared by both oracles (2 layers: 2-2.4 G parameters)
    sd = {k: synth.synth_bf16(seed, *v) for k, v in specs.items()}
    make32 = lambda: Ref(cfg, sd, torch.float32)
    makebf = lambda: Ref(cfg, sd, torch.bfloat16)
    d = _model_dir(tmp_path, cfg)
    p1 = _prompts(cfg["vocab_size"], (61,), 100)
    p8 = _prompts(cfg["vocab_size"], LENS8, 200)
    # (tag, params, prompts, persistent kernel?); Falcon has no persistent kernel
    runs = [("b1", {}, p1, not falcon), ("b8 wgmma", {}, p8, False)]
    if not falcon:
        runs.insert(1, ("b1 multi-kernel gemv (the per-rank path under tensor parallelism)", {"use_mega": 0}, p1, False))
        # the persistent kernel's batched instantiations on ragged rows: 4 rows at 7B; at 70B (K = 28672) 4 rows of staged
        # activations do not fit its shared memory next to the ring, so the largest batch it takes there is 2.  The
        # synthetic full-width logits are near-flat: at about one position in five the fp32 oracle's top-2 margin is below
        # the bf16 noise, where either id is a valid pick.  The 7B rows are batch-8 prompts with few such positions (3 of
        # 20; the CPU bf16 oracle itself picks another id at one), so that the exact-id count stays meaningful.
        nb = 2 if cfg["intermediate_size"] > 16384 else 4
        pb = [p8[i] for i in (0, 3, 5, 6)] if nb == 4 else _prompts(cfg["vocab_size"], (44, 70), 300)
        runs.append((f"b{nb} persistent kernel", {"mega_max_batch": 4}, pb, True))
    for tag, mode, prompts, mega in runs:
        with Engine(d, dict(mode, weights="synthetic", seed=seed, max_batch=8, max_seq_len=128)) as e:
            toks, lg, launches = generate_counted(e, prompts, 5, want_logits=True)
        assert_decode_path(launches, 4, mega, f"{name} {tag}")
        assert np.isfinite(lg).all()
        check_against_oracle(f"{name} L=2 {tag}", make32, makebf, prompts, toks, lg)


def _write_random_q4_0_gguf(path, cfg, seed):
    """A well-formed Q4_0 GGUF at cfg's shapes with random blocks (random nibbles, fp16 scale ~ W_AMP/8): llama.cpp's
    container and tensor naming (convert_hf_to_gguf), q/k rows in llama.cpp's permuted order.  Returns the HF-layout
    bf16 state dict of gguf-py's own dequantisation (the oracle's weights)."""
    from gguf import GGMLQuantizationType as T
    from gguf import GGUFWriter, quants

    rng = np.random.default_rng(seed)
    w = GGUFWriter(path, "llama")
    h, nh, nkv = cfg["hidden_size"], cfg["num_attention_heads"], cfg["num_key_value_heads"]
    w.add_context_length(cfg["max_position_embeddings"])
    w.add_embedding_length(h)
    w.add_block_count(cfg["num_hidden_layers"])
    w.add_feed_forward_length(cfg["intermediate_size"])
    w.add_head_count(nh)
    w.add_head_count_kv(nkv)
    w.add_layer_norm_rms_eps(cfg["rms_norm_eps"])
    w.add_rope_freq_base(cfg["rope_theta"])
    names = {"self_attn.q_proj": "attn_q", "self_attn.k_proj": "attn_k", "self_attn.v_proj": "attn_v",
             "self_attn.o_proj": "attn_output", "mlp.gate_proj": "ffn_gate", "mlp.up_proj": "ffn_up",
             "mlp.down_proj": "ffn_down", "input_layernorm": "attn_norm", "post_attention_layernorm": "ffn_norm"}
    deq = {}
    for k, (_tid, shape, amp, base) in synth.llama_tensor_specs(cfg).items():
        if k == "model.embed_tokens.weight":
            g = "token_embd.weight"
        elif k == "model.norm.weight":
            g = "output_norm.weight"
        elif k == "lm_head.weight":
            g = "output.weight"
        else:
            _, _, l, rest = k.split(".", 3)
            g = f"blk.{l}." + names[rest.rsplit(".", 1)[0]] + ".weight"
        if len(shape) == 2:
            rows, cols = shape
            nb = cols // 32
            raw = rng.integers(0, 256, size=(rows, nb, 18), dtype=np.uint8)
            dscale = (amp / 8.0 * (0.5 + rng.random((rows, nb), dtype=np.float32))).astype(np.float16)
            raw[:, :, 0:2] = dscale.view(np.uint8).reshape(rows, nb, 2)
            raw = raw.reshape(rows, nb * 18)
            w.add_tensor(g, raw, raw_dtype=T.Q4_0)
            dq = quants.dequantize(raw, T.Q4_0)
            if "q_proj" in k or "k_proj" in k:  # file order is llama.cpp's permuted order: undo it for the HF-layout oracle
                heads = nh if "q_proj" in k else nkv
                dq = dq.reshape(heads, dq.shape[0] // heads // 2, 2, *dq.shape[1:]).swapaxes(1, 2).reshape(dq.shape)
            deq[k] = torch.from_numpy(np.ascontiguousarray(dq)).to(torch.bfloat16)
        else:
            a = (base + amp * (2 * rng.random(shape, dtype=np.float32) - 1)).astype(np.float32)
            w.add_tensor(g, a)
            deq[k] = torch.from_numpy(a).to(torch.bfloat16)
    w.write_header_to_file()
    w.write_kv_data_to_file()
    w.write_tensors_to_file()
    w.close()
    return deq


def test_true_width_13b_from_q4_0_gguf(tmp_path):
    """BASELINE config 3 at its true width: a 2-layer Llama-2-13B-shaped Q4_0 GGUF `model.bin` (0.54 GB) goes through the
    GGUF reader + dequant-on-load kernel into the bf16 engine; the oracle runs on gguf-py's dequantisation of the same
    blocks.  Batch 1 and batch 8."""
    pytest.importorskip("gguf")
    from substratus_b200 import Engine

    cfg = dict(synth.LLAMA2_13B, num_hidden_layers=2)
    deq = _write_random_q4_0_gguf(str(tmp_path / "model.bin"), cfg, 7)
    make32 = lambda: llama_ref.LlamaRef(cfg, deq, torch.float32)
    makebf = lambda: llama_ref.LlamaRef(cfg, deq, torch.bfloat16)
    p1 = _prompts(cfg["vocab_size"], (61,), 101)
    p8 = _prompts(cfg["vocab_size"], LENS8, 201)
    with Engine(str(tmp_path), {"max_batch": 8, "max_seq_len": 128}) as e:
        assert e.info.hidden_size == 5120 and e.info.n_layers == 2
        for tag, prompts in (("b1", p1), ("b8 wgmma", p8)):
            toks, lg = e.generate(prompts, 5, want_logits=True)
            check_against_oracle(f"llama2-13b Q4_0 GGUF L=2 {tag}", make32, makebf, prompts, toks, lg)


def test_full_depth_7b_vs_fp32_oracle(tmp_path):
    """All 32 layers of Llama-2-7B (BASELINE configs[1], the headline workload) against the fp32 oracle: one 24-token
    prompt, first-token logits + 4 decode steps, persistent decode kernel.  The oracles stream their weights tensor by
    tensor (oracle.synth.LazyStateDict), so the fp32 truth never holds 27 GB."""
    from substratus_b200 import Engine

    cfg = dict(synth.LLAMA2_7B)
    seed = 0
    specs = synth.llama_tensor_specs(cfg)
    make32 = lambda: llama_ref.LlamaRef(cfg, synth.LazyStateDict(specs, seed, torch.float32), torch.float32)
    makebf = lambda: llama_ref.LlamaRef(cfg, synth.LazyStateDict(specs, seed, torch.bfloat16), torch.bfloat16)
    prompts = _prompts(cfg["vocab_size"], (24,), 1234)
    with Engine(_model_dir(tmp_path, cfg), {"weights": "synthetic", "seed": seed, "max_batch": 2, "max_seq_len": 128}) as e:
        toks, lg, launches = generate_counted(e, prompts, 5, want_logits=True)
    assert_decode_path(launches, 4, True, "llama2-7b L=32 b1")
    check_against_oracle("llama2-7b L=32 b1 persistent kernel", make32, makebf, prompts, toks, lg)
