"""Shared helpers for the parity tests."""
import json
import os

import numpy as np

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def load_gold(name):
    with open(os.path.join(GOLD, name + ".json")) as f:
        return json.load(f)


def greedy_agree(tok_a, tok_b, logits_b, eps):
    """Greedy sequences tok_a / tok_b ([nseq, n]) agree if, per sequence, they are identical up to the first step
    where they differ AND at that step the reference logits (logits_b [nseq, n, V], the logits tok_b was picked
    from) separate the two candidates by less than eps (a rounding-level tie); after a tie the sequences follow
    different contexts and are not compared.  Returns (ok, n_exact_steps_total, message)."""
    tok_a = np.asarray(tok_a)
    tok_b = np.asarray(tok_b)
    exact = 0
    for i in range(tok_a.shape[0]):
        for s in range(tok_a.shape[1]):
            if tok_a[i, s] == tok_b[i, s]:
                exact += 1
                continue
            gap = float(logits_b[i, s, tok_b[i, s]] - logits_b[i, s, tok_a[i, s]])
            if gap >= eps:
                return False, exact, f"seq {i} step {s}: {tok_a[i, s]} vs {tok_b[i, s]} with margin {gap:.4g} >= {eps}"
            break
    return True, exact, "ok"


def rel_err(a, ref):
    """SURVEY.md §7 metric: max|a-ref| / max|ref|."""
    a = np.asarray(a, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    return float(np.abs(a - ref).max() / np.abs(ref).max())


def generate_counted(e, prompts, max_new_tokens, want_logits=False):
    """Engine.generate, plus the kernel launches of its decode steps: the witness of which decode path ran.  The
    persistent kernel is one launch per step (Engine::forward_mega); the graph and stream paths launch every kernel of
    the multi-kernel forward, several per layer.  Returns (tokens [nseq, n], logits [n, nseq, V] or None, launches)."""
    assert max_new_tokens >= 2
    sids = [e.seq_create() for _ in prompts]
    try:
        first, lg0 = e.prefill(sids, prompts, want_logits)
        e.timing_reset()
        rest, lg = e.decode(sids, first, max_new_tokens - 1, want_logits)
        launches = e.timing().kernel_launches
        toks = np.concatenate([first[:, None], rest], axis=1)
        return toks, (np.concatenate([lg0[None], lg], axis=0) if want_logits else None), launches
    finally:
        for s in sids:
            e.seq_free(s)


def assert_decode_path(launches, n_steps, mega, what=""):
    """The witness: n_steps decode steps ran on the persistent kernel (mega) or on the multi-kernel path (not mega)."""
    if mega:
        assert launches == n_steps, f"{what}: {launches} kernel launches for {n_steps} decode steps: not the persistent kernel"
    else:
        assert launches > n_steps, f"{what}: {launches} kernel launches for {n_steps} decode steps: not the multi-kernel path"


def oracle_logits(make_ref, prompts, toks):
    """[nseq, n, V] fp32 logits of one oracle for every position the engine picked a token at, teacher-forced with the
    engine's own picks: ONE pass per sequence over prompt + toks[:-1]."""
    import torch

    out = []
    ref = make_ref()
    for p, t in zip(prompts, toks):
        ref.reset()
        ids = torch.tensor([list(p) + [int(x) for x in t[:-1]]])
        out.append(ref.forward(ids)[0, len(p) - 1:].float().numpy())
    del ref
    return np.stack(out)


def check_against_oracle(what, make32, makebf, prompts, toks, lg, diag=print, tol=1e-3):
    """Every position the engine produced logits for, against the fp32 oracle (truth) and the bf16 oracle (noise
    yardstick), both teacher-forced with the engine's own ids.  toks [nseq, n], lg [n, nseq, V] from the engine.
    err = max|x - fp32| / max|fp32| per position; the engine's error must be within tol of the bf16 oracle's on the mean,
    with the slack of two independent noise draws at the extremes (tests/test_parity_gpu.py::_assert_parity).  Every
    greedy id must be the fp32 argmax unless the oracle's margin is below 4 x its own bf16 noise (a rounding-level tie),
    and ties are the exception.  Returns the measured (mean err_gpu, mean err_cpu)."""
    import time

    lg = np.transpose(lg, (1, 0, 2))
    t0 = time.time()
    l32 = oracle_logits(make32, prompts, toks)
    lbf = oracle_logits(makebf, prompts, toks)
    n = toks.shape[1]
    eg = np.array([[rel_err(lg[i, s], l32[i, s]) for s in range(n)] for i in range(len(prompts))])
    ec = np.array([[rel_err(lbf[i, s], l32[i, s]) for s in range(n)] for i in range(len(prompts))])
    noise = 4 * float(np.abs(lbf - l32).max())
    exact, ties = 0, 0
    for i in range(len(prompts)):
        for s in range(n):
            want = int(l32[i, s].argmax())
            if want == int(toks[i, s]):
                exact += 1
                continue
            gap = float(l32[i, s, want] - l32[i, s, toks[i, s]])
            assert gap < noise, f"{what}: seq {i} step {s}: engine picked {toks[i, s]}, fp32 oracle {want} with margin {gap:.4g} >= noise {noise:.4g}"
            ties += 1
    diag(f"[{what}] err_gpu mean {eg.mean():.3e} max {eg.max():.3e} | err_cpu_bf16 mean {ec.mean():.3e} max {ec.max():.3e} | "
         f"positions {eg.size} | greedy ids == fp32 oracle argmax: {exact}/{eg.size} (+{ties} rounding-level ties, eps {noise:.3e}) | oracle {time.time() - t0:.1f}s")
    assert eg.mean() <= ec.mean() + tol, (what, eg.mean(), ec.mean())
    assert eg.max() <= 1.5 * ec.max() + tol, (what, eg.max(), ec.max())
    assert (eg <= 2 * ec + tol).all(), (what, eg, ec)
    assert exact >= eg.size - max(1, eg.size // 8), (what, exact, eg.size)  # ties are the exception, not the rule
    return float(eg.mean()), float(ec.mean())


def assert_greedy_valid(cfg, sd, prompts, toks, what=""):
    """Every id in toks[i] must be a valid greedy pick for ITS OWN context: the fp32 oracle, teacher-forced with the ids
    under test, must either pick the same id or separate the two candidates by less than the bf16 noise (4 x the largest
    bf16-vs-fp32 logit difference of the oracle itself).  Unlike comparing with a solo run, this holds however batch-mates
    change the GEMM schedule.  Returns the number of exact matches."""
    import torch

    from oracle import llama_ref

    exact = 0
    r32 = llama_ref.LlamaRef(cfg, sd, torch.float32)
    rbf = llama_ref.LlamaRef(cfg, sd, torch.bfloat16)
    for p, t in zip(prompts, toks):
        ids = torch.tensor([list(p) + [int(x) for x in t[:-1]]])
        r32.reset()
        rbf.reset()
        l32 = r32.forward(ids)[0, len(p) - 1:].float().numpy()
        lbf = rbf.forward(ids)[0, len(p) - 1:].float().numpy()
        noise = 4 * float(np.abs(lbf - l32).max())
        for s_, tok in enumerate(t):
            want = int(l32[s_].argmax())
            if want == int(tok):
                exact += 1
                continue
            gap = float(l32[s_, want] - l32[s_, int(tok)])
            assert gap < noise, f"{what}: prompt len {len(p)} step {s_}: got {tok}, fp32 oracle picks {want} with margin {gap:.4g} >= noise {noise:.4g}"
    return exact
