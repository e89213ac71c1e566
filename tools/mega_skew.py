"""Per-phase arrival skew of the persistent decode kernel across ALL CTAs (params.mega_prof = 2): for every stamp of the
phase timeline, the spread (last CTA - first CTA) and which SMs are systematically late.  Usage:
    python tools/mega_skew.py [workload=llama2-7b] [batch=1]"""
import json, os, sys, tempfile
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from substratus_b200 import Engine
import bench

wl = sys.argv[1] if len(sys.argv) > 1 else "llama2-7b"
B = int(sys.argv[2]) if len(sys.argv) > 2 else 1
cfg = bench.WORKLOADS[wl]
d = tempfile.mkdtemp()
json.dump(cfg, open(os.path.join(d, "config.json"), "w"))
extra = json.loads(sys.argv[3]) if len(sys.argv) > 3 else {}
e = Engine(d, dict({"weights": "synthetic", "max_batch": 4, "max_seq_len": 700, "mega_prof": 2}, **extra))
rng = np.random.default_rng(0)
prompts = [rng.integers(0, cfg["vocab_size"], 512).tolist() for _ in range(B)]
sids = [e.seq_create() for _ in range(B)]
nxt, _ = e.prefill(sids, prompts)
out, _ = e.decode(sids, nxt, 16)  # warm-up call
e.decode(sids, out[:, -1], 16)
t = e.debug_read("mega_prof_all")           # [n_ctas, 1024] us, -1 = unset; col 1023 = smid
smid = t[:, 1023].astype(int)
L = cfg["num_hidden_layers"]
n = min(1 + 14 * L, 1022)
T = t[:, :n]
names = ["stage_x(qkv)", "qkv", "sync1", "attn", "sync2", "stage_x(o)", "o", "sync3", "stage_x(gu)", "gate_up", "sync4", "stage_x(down)", "down", "sync5"]
nl = (n - 1) // 14
per = T[:, 1:1 + 14 * nl].reshape(T.shape[0], nl, 14)      # stamp k of layer l = END of phase k
print(f"{wl} B={B}: {T.shape[0]} CTAs, {nl} layers profiled; step total {T[:, :n].max():.1f} us")
# arrival = stamp just BEFORE each sync (end of the preceding phase); the sync ends when the last CTA arrives
print("phase end           mean duration(CTA-avg)   spread last-first (mean over layers)   p50 lateness of the 8 latest SMs")
prev = np.concatenate([T[:, :1, None].repeat(1, 1), per[:, :-1, 13:14]], axis=1)[:, :, 0]  # start of each layer per CTA
for k in range(14):
    end = per[:, 2:, k]
    start = per[:, 2:, k - 1] if k > 0 else prev[:, 2:]
    dur = (end - start).mean()
    spread = (end.max(0) - end.min(0)).mean()
    print(f"  {names[k]:14s} {dur:8.2f} us   spread {spread:6.2f} us")
# systematic lateness per CTA at the arrival stamps of the weight phases (qkv=1, o=6, gate_up=9, down=12)
late = np.zeros(T.shape[0])
for k in (1, 6, 9, 12):
    end = per[:, 2:, k]
    late += (end - end.min(0, keepdims=True)).mean(1)
order = np.argsort(-late)
print("latest CTAs (sum over the 4 weight phases of mean lateness vs the first arriver, us): ")
print("  " + ", ".join(f"cta{c}/sm{smid[c]}:{late[c]:.1f}" for c in order[:10]))
print("earliest: " + ", ".join(f"cta{c}/sm{smid[c]}:{late[c]:.1f}" for c in order[-6:]))
print(f"lateness: mean {late.mean():.2f} std {late.std():.2f} max {late.max():.2f} us per layer")
dur = sum((per[:, 2:, k] - per[:, 2:, k - 1]).mean(1) for k in (1, 6, 9, 12))
print(f"weight-phase time per CTA and layer: min {dur.min():.1f} median {np.median(dur):.1f} max {dur.max():.1f} us "
      "(passes are claimed at run time, so a slow SM streams fewer of them)")
np.save(os.path.join("gpurun_out", f"mega_skew_{wl}_b{B}.npy"), t) if os.path.isdir("gpurun_out") else None
