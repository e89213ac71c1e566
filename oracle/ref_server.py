"""TEST INFRASTRUCTURE — the reference's CPU serving container, restated (BASELINE config 1:
"examples/facebook-opt-125m greedy decode, 1 request, reference CPU container (plumbing, no GPU)").

The reference serves `examples/facebook-opt-125m/base-server.yaml` with the external image
`substratusai/model-server-basaran` (Basaran = HF transformers behind an OpenAI-style `/v1/completions`); that image
is not in the tree and cannot be pulled offline.  This module is the same plumbing on the library the image wraps:
HF `AutoModelForCausalLM` on CPU behind the SAME container contract the serve host honours
(docs/container-contract.md:50-55: port 8080, `GET /` -> 200 when ready; the only request the reference sends is
`POST /v1/completions {"prompt", "max_tokens"}`, test/system.sh:73-78).  It lets the tests and bench.py drive both
servers through one client.  Prompts are token-id arrays (no tokenizer files exist offline).

    python -m oracle.ref_server --model-dir /content/model --port 8080
"""
from __future__ import annotations

import argparse
import json
import threading
import time
from http.server import BaseHTTPRequestHandler, ThreadingHTTPServer


class State:
    model = None
    ready = False
    lock = threading.Lock()


def load(model_dir: str, dtype: str = "bfloat16"):
    import torch
    from transformers import AutoConfig, AutoModelForCausalLM

    cfg = AutoConfig.from_pretrained(model_dir)
    try:
        m = AutoModelForCausalLM.from_pretrained(model_dir, dtype=getattr(torch, dtype))
    except Exception:  # config-only directory: random init at the config's shapes (no checkpoints exist offline)
        torch.manual_seed(0)
        m = AutoModelForCausalLM.from_config(cfg).to(getattr(torch, dtype))
    State.model = m.eval()
    State.ready = True


class Handler(BaseHTTPRequestHandler):
    def log_message(self, *a):
        pass

    def _send(self, code, obj):
        body = json.dumps(obj).encode()
        self.send_response(code)
        self.send_header("Content-Type", "application/json")
        self.send_header("Content-Length", str(len(body)))
        self.end_headers()
        self.wfile.write(body)

    def do_GET(self):
        if self.path.split("?")[0] in ("/", "/healthz"):
            self._send(200 if State.ready else 503, {"status": "ready" if State.ready else "loading"})
        else:
            self._send(404, {"error": "no such endpoint"})

    def do_POST(self):
        import torch

        path = self.path.split("?")[0]
        if path not in ("/v1/completions", "/generate"):
            return self._send(404, {"error": "no such endpoint"})
        if not State.ready:
            return self._send(503, {"error": "model is not loaded yet"})
        try:
            req = json.loads(self.rfile.read(int(self.headers.get("Content-Length", "0"))) or b"{}")
            ids = req.get("prompt" if path == "/v1/completions" else "tokens")
            n = int(req.get("max_tokens" if path == "/v1/completions" else "max_new_tokens", 16))
            if not isinstance(ids, list) or not ids or not all(isinstance(t, int) for t in ids):
                return self._send(400, {"error": "pass the prompt as an array of token ids"})
        except Exception as ex:
            return self._send(400, {"error": str(ex)})
        with State.lock, torch.no_grad():
            t0 = time.time()
            x = torch.tensor([ids])
            out = State.model(x, use_cache=True)
            nxt = out.logits[:, -1].float().argmax(-1)
            ttft = time.time() - t0
            toks, past = [int(nxt)], out.past_key_values
            for _ in range(n - 1):
                out = State.model(nxt[:, None], past_key_values=past, use_cache=True)
                past = out.past_key_values
                nxt = out.logits[:, -1].float().argmax(-1)
                toks.append(int(nxt))
            dec = time.time() - t0 - ttft
        extra = {"ttft_ms": ttft * 1e3, "decode_ms": dec * 1e3,
                 "decode_tokens_per_sec": (n - 1) / dec if n > 1 and dec > 0 else 0.0}
        if path == "/generate":
            self._send(200, dict({"tokens": toks}, **extra))
        else:
            self._send(200, dict({"object": "text_completion", "choices": [{"index": 0, "text": "", "tokens": toks,
                                                                           "finish_reason": "length"}],
                                  "usage": {"prompt_tokens": len(ids), "completion_tokens": len(toks)}}, **extra))


def serve(model_dir: str, port: int, dtype: str = "bfloat16"):
    State.ready, State.model = False, None  # a second server in one process must not answer with the previous model
    srv = ThreadingHTTPServer(("0.0.0.0", port), Handler)
    threading.Thread(target=load, args=(model_dir, dtype), daemon=True).start()
    return srv


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--model-dir", default="/content/model")
    ap.add_argument("--port", type=int, default=8080)
    ap.add_argument("--dtype", default="bfloat16")
    a = ap.parse_args()
    serve(a.model_dir, a.port, a.dtype).serve_forever()
