"""Per-kernel-class bandwidth of the decode projections at Llama-2-7B shapes (HBM-streamed vs L2-resident)."""
import json, os, sys, tempfile
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import synth
from substratus_b200 import Engine
mode = json.loads(sys.argv[1]) if len(sys.argv) > 1 else {}
rows = int(sys.argv[2]) if len(sys.argv) > 2 else 1
d = tempfile.mkdtemp()
json.dump(synth.LLAMA2_7B, open(os.path.join(d, "config.json"), "w"))
e = Engine(d, dict(mode, weights="synthetic", max_batch=max(4, rows), max_seq_len=700))
for k in ("o", "o@l2", "qkv", "qkv@l2", "down", "down@l2", "gate_up", "lm_head", "attn"):
    ms, by = e.bench_kernel(k, rows=rows, ctx=576, iters=128)
    print(f"{k:10s} {ms*1e3:8.2f} us  {by/ms/1e6:8.1f} GB/s  ({by/ms/1e6/132:6.1f} GB/s/SM)", flush=True)
