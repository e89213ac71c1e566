"""CPU suite (-m "not gpu"): pins the oracle restatement to HF transformers and the golden vectors,
checks the host twin of the synthetic generator, and that the C-ABI library loads with every
symbol include/ssb.h declares (no compute without a GPU: the engine must refuse, not fall back)."""
import json
import os
import re

import numpy as np
import pytest
import torch

from oracle import llama_ref, synth

from util import GOLD, greedy_agree, load_gold, rel_err


@pytest.mark.parametrize("name", ["tiny_mha", "tiny_gqa"])
def test_oracle_matches_golden(name):
    """Restatement (oracle/llama_ref.py) reproduces the committed HF outputs.  On the CPU that generated the
    vectors this is bit-for-bit; oneDNN may pick other bf16 kernels on another CPU, so the pin is: fp32 logits
    within 1e-4 absolute, bf16 logits within one bf16 ulp of the largest logit, greedy ids equal up to
    rounding-level ties (tests/util.py::greedy_agree)."""
    g = load_gold(name)
    sd = synth.llama_state_dict(g["config"], g["weight_seed"])
    assert int(sum(int(v.view(torch.int16).to(torch.int64).sum()) for v in sd.values())) == g["weights_checksum"]
    ids = torch.tensor(g["prompt"])
    for tag, dt in (("bf16", torch.bfloat16), ("fp32", torch.float32)):
        ref = llama_ref.LlamaRef(g["config"], sd, dt)
        toks, lg = ref.generate(ids, g["max_new_tokens"])
        want = torch.tensor(g[f"first_logits_{tag}"])
        tol = 2.0 ** -7 * float(want.abs().max()) if dt == torch.bfloat16 else 1e-4
        assert (lg[:, 0] - want).abs().max().item() <= tol
        ok, exact, msg = greedy_agree(g[f"tokens_{tag}"], toks.numpy(), lg.numpy(), 4 * tol + 1e-6)
        assert ok, msg
        assert exact >= toks.shape[1]  # at least one sequence's worth of exactly equal picks


def test_oracle_matches_hf_live():
    """Same check against HF imported live (it ships in the image on both boxes), other seed/shape."""
    cfg = dict(synth.TINY_GQA, num_hidden_layers=2, vocab_size=640)
    sd = synth.llama_state_dict(cfg, 11)
    ids = torch.randint(0, cfg["vocab_size"], (3, 9), generator=torch.Generator().manual_seed(5))
    for dt in (torch.bfloat16, torch.float32):
        hf = llama_ref.hf_model(cfg, sd, dt)
        with torch.no_grad():
            want = hf(ids).logits
        got = llama_ref.LlamaRef(cfg, sd, dt).forward(ids)
        assert torch.equal(got, want)


def test_falcon_oracle_matches_hf_live():
    """oracle/falcon_ref.py == HF FalconForCausalLM (eager, new decoder architecture) bit-for-bit, bf16 and fp32,
    for GQA (kv=2) and MQA-like (kv=1) groupings, forward and greedy generation."""
    from oracle import falcon_ref as fr

    for kv in (2, 1):
        cfg = dict(fr.TINY_FALCON, num_kv_heads=kv)
        sd = fr.falcon_state_dict(cfg, 5)
        ids = torch.randint(0, cfg["vocab_size"], (2, 13), generator=torch.Generator().manual_seed(1))
        for dt in (torch.bfloat16, torch.float32):
            hf = fr.hf_model(cfg, sd, dt)
            with torch.no_grad():
                want = hf(ids).logits
                out = hf.generate(ids, max_new_tokens=5, do_sample=False, pad_token_id=0)[:, 13:]
            assert torch.equal(fr.FalconRef(cfg, sd, dt).forward(ids), want)
            assert torch.equal(fr.FalconRef(cfg, sd, dt).generate(ids, 5)[0], out)


def test_oracle_incremental_equals_full():
    """KV-cache decode of the restatement equals a full re-forward (property the CUDA path is also held to)."""
    cfg = synth.TINY_MHA
    sd = synth.llama_state_dict(cfg, 1)
    ids = torch.randint(0, cfg["vocab_size"], (1, 12), generator=torch.Generator().manual_seed(2))
    ref = llama_ref.LlamaRef(cfg, sd, torch.float32)
    full = ref.forward(ids)[:, -1]
    ref.reset()
    ref.forward(ids[:, :8])
    for t in range(8, 12):
        last = ref.forward(ids[:, t:t + 1])[:, -1]
    assert (last - full).abs().max().item() < 1e-4


def test_synth_host_twin_bit_exact(lib):
    """C++ host twin of the synthetic generator == numpy oracle (the CUDA twin is checked in the gpu suite)."""
    from substratus_b200 import synth_fill_host

    for seed, tid, start, n, amp, base in [(0, 0, 0, 4096, synth.W_AMP, 0.0), (7, 35, 12345, 1000, synth.NORM_AMP, 1.0),
                                           (3, synth.GLOBAL + 2, 2 ** 33, 512, synth.W_AMP * synth.LMHEAD_GAIN, 0.0)]:
        got = synth_fill_host(seed, tid, start, n, amp, base)
        want = synth.f32_to_bf16_bits(synth.synth_f32(seed, tid, n, amp, base, start))
        assert np.array_equal(got, want)


def test_abi_exports_every_declared_symbol(lib):
    hdr = open(os.path.join(os.path.dirname(GOLD), "..", "include", "ssb.h")).read()
    declared = set(re.findall(r"\b(ssb_[a-z0-9_]+)\s*\(", hdr))
    declared -= {"ssb_engine", "ssb_info", "ssb_timing"}
    from substratus_b200.engine import EXPORTS

    assert declared == set(EXPORTS), declared ^ set(EXPORTS)
    for s in declared:
        assert getattr(lib, s) is not None


def test_no_cpu_fallback(lib, tmp_path):
    """Without an sm_90 device engine creation must fail loudly (SSB_ENODEV), never compute on the CPU."""
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from substratus_b200 import Engine, SsbError

    llama_ref.write_hf_dir(str(tmp_path), synth.TINY_MHA, {})
    with pytest.raises(SsbError) as ei:
        Engine(str(tmp_path), {"weights": "synthetic"})
    assert ei.value.code == -3, ei.value


def test_bad_inputs_rejected(lib, tmp_path):
    from substratus_b200 import Engine, SsbError

    with pytest.raises(SsbError):
        Engine(str(tmp_path / "nope"), {})
    (tmp_path / "config.json").write_text("{not json")
    with pytest.raises(SsbError):
        Engine(str(tmp_path), {})
    with pytest.raises(SsbError):
        Engine(str(tmp_path), None and {} or {"x": 1}, None) if False else Engine(str(tmp_path), {"weights": "synthetic"})
