"""Phase timeline of the persistent decode kernel (CTA 0) at Llama-2-7B shapes: prints per-phase microseconds averaged
over the layers."""
import json, os, sys, tempfile
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from oracle import synth
from substratus_b200 import Engine
B = int(sys.argv[1]) if len(sys.argv) > 1 else 1
CFG = {"llama2-7b": synth.LLAMA2_7B, "llama2-13b": synth.LLAMA2_13B, "llama2-70b": synth.LLAMA2_70B}[sys.argv[2] if len(sys.argv) > 2 else "llama2-7b"]
d = tempfile.mkdtemp()
json.dump(CFG, open(os.path.join(d, "config.json"), "w"))
e = Engine(d, {"weights": "synthetic", "max_batch": 4, "max_seq_len": 700, "mega_prof": 1})
rng = np.random.default_rng(0)
prompts = [rng.integers(0, 32000, 512).tolist() for _ in range(B)]
sids = [e.seq_create() for _ in range(B)]
nxt, _ = e.prefill(sids, prompts)
e.decode(sids, nxt, 64)
t = e.debug_read("mega_prof")[0]
L = min(CFG["num_hidden_layers"], (1023 - 1) // 14)
per = t[1:1 + 14 * L].reshape(L, 14)
prev = np.concatenate([[t[0]], per[:-1, 13]])
names = ["stage_x(qkv)", "qkv", "sync", "attn", "sync", "stage_x(o)", "o", "sync", "stage_x(gu)", "gate_up", "sync", "stage_x(down)", "down", "sync"]
d_ = np.diff(np.concatenate([prev[:, None], per], axis=1), axis=1)
print("step total us:", t[-1], " per layer mean us:", d_.sum(1).mean())
for n, v, s in zip(names, d_[2:].mean(0), d_[2:].std(0)):
    print(f"  {n:14s} {v:7.2f} us  (std {s:.2f})")
print("timing decode_ms/64 =", e.timing().decode_ms / 64)
