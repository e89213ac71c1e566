"""Writes the ids and fp32 logits of one fixed tiny-model generation to an .npz — run once on the parent and once on the
change and compare with tools/ab_bitexact.py (a change that does not touch the arithmetic must be bit-identical)."""
import os, sys, tempfile
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from oracle import llama_ref, synth
from substratus_b200 import Engine

out = sys.argv[1]
cfg = synth.TINY_GQA
d = tempfile.mkdtemp()
llama_ref.write_hf_dir(d, cfg, synth.llama_state_dict(cfg, 21))
g = torch.Generator().manual_seed(3)
res = {}
for name, prompts in (("b1", [torch.randint(0, cfg["vocab_size"], (37,), generator=g).tolist()]),
                      ("b3", [torch.randint(0, cfg["vocab_size"], (n,), generator=g).tolist() for n in (5, 18, 64)]),
                      # 12 rows: tensor-core stream-K decode projections (tc_min_rows = 8) and the split-context attention kernels
                      ("b12", [torch.randint(0, cfg["vocab_size"], (n,), generator=g).tolist() for n in range(3, 39, 3)])):
    with Engine(d, {"max_batch": 16, "max_seq_len": 160}) as e:
        toks, lg = e.generate(prompts, 12, want_logits=True)
    res[name + "_toks"], res[name + "_logits"] = toks, lg
np.savez(out, **res)
print("wrote", out)
