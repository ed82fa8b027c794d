#!/usr/bin/env python
"""Evaluate a Llama model with per-token log-likelihoods (``LlamaForCausalLM.score``); prints one JSON object.

    # held-out perplexity on pre-tokenised shards (seeded windows of --seq-len tokens)
    python scripts/evaluate.py --model 150m --checkpoint outputs/model_step_1000 --weights outer \\
        --tokens "/data/c4-val/*.tok" --seq-len 1024 --batch-size 8 --batches 50
    # multiple choice: one request per line, {"context": [ids], "choices": [[ids], ...], "gold": k}
    python scripts/evaluate.py --model /models/llama-150m --choices hellaswag.jsonl

The model is chosen as in scripts/generate.py: an HF directory, a preset, or a train_fsdp checkpoint with
``--weights local|outer``.

Perplexity reports ``loss`` (mean negative log-likelihood per scored token; the first token of a window is not scored),
``perplexity`` = exp(loss), ``tokens`` (scored) and ``tokens_per_s`` (window tokens through ``score`` per second).
Multiple choice scores each choice by the sum of its continuation log-probabilities given the context and reports
``acc`` (argmax of the sum), ``acc_per_token`` (argmax of the sum over the continuation length in tokens), ``greedy``
(fraction of gold continuations that are the greedy continuation at every token) and ``n`` (requests).  Requests are
sorted by length and scored in right-padded batches of --batch-size sequences.  ``context`` and ``choices`` may also be
text when a local ``--tokenizer`` directory is given.

``--fp8-weights`` scores the model with its decoder-layer projections quantised to e4m3, one scale per output row (what
``generate.py --fp8-weights`` decodes with), and adds ``"fp8_weights": true`` to the result: compare it with a run
without the flag to see what the quantisation costs.
"""
import argparse
import json
import math
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from generate import add_model_args, load_model  # noqa: E402


def _sync(device: torch.device) -> None:
    if device.type == "cuda":
        torch.cuda.synchronize(device)


def perplexity(model, pattern: str, seq_len: int, batch_size: int, batches: int, seed: int, fp8_weights: bool = False) -> dict:
    from opendiloco_b200.utils.data import TokenFileLoader

    dev = model.device
    loader = TokenFileLoader(pattern, batch_size, seq_len, seed=seed, pin_memory=False)
    try:
        nll, n_tok, seconds = 0.0, 0, 0.0
        for _ in range(batches):
            ids = next(loader)["input_ids"].to(dev)
            _sync(dev)
            t0 = time.perf_counter()
            lp = model.score(ids, fp8_weights=fp8_weights).logprobs
            _sync(dev)
            seconds += time.perf_counter() - t0
            nll -= float(lp[:, 1:].double().sum())
            n_tok += ids.shape[0] * (ids.shape[1] - 1)
    finally:
        loader.close()
    loss = nll / n_tok
    return {"loss": loss, "perplexity": math.exp(loss), "tokens": n_tok,
            "tokens_per_s": batches * batch_size * seq_len / seconds}


def _ids(x, tok, what: str, special: bool) -> list[int]:
    if isinstance(x, str):
        if tok is None:
            raise SystemExit(f"error: {what} is text; give --tokenizer or token ids")
        return list(tok(x, add_special_tokens=special)["input_ids"])
    return [int(t) for t in x]


def multiple_choice(model, path: str, batch_size: int, tok, fp8_weights: bool = False) -> dict:
    requests = []
    with open(path) as f:
        for n, line in enumerate(f, 1):
            if not line.strip():
                continue
            r = json.loads(line)
            ctx = _ids(r["context"], tok, f"line {n} context", True)
            choices = [_ids(c, tok, f"line {n} choice", False) for c in r["choices"]]
            if not ctx or not choices or any(not c for c in choices):
                raise SystemExit(f"error: line {n}: the context and every choice need at least one token")
            gold = int(r["gold"])
            if not 0 <= gold < len(choices):
                raise SystemExit(f"error: line {n}: gold {gold} is not a choice index")
            requests.append((ctx, choices, gold))
    if not requests:
        raise SystemExit(f"error: {path} holds no requests")
    # one sequence per (request, choice); sorted by length so that a batch needs little padding
    seqs = [(len(ctx) + len(c), q, k) for q, (ctx, choices, _) in enumerate(requests) for k, c in enumerate(choices)]
    seqs.sort()
    total = {}                                         # (request, choice) -> (sum of logprobs, all greedy)
    dev = model.device
    for b0 in range(0, len(seqs), batch_size):
        batch = seqs[b0:b0 + batch_size]
        S = batch[-1][0]
        ids = torch.zeros(len(batch), S, dtype=torch.int64)
        mask = torch.zeros(len(batch), S, dtype=torch.int64)
        for i, (n, q, k) in enumerate(batch):
            ctx, choices, _ = requests[q]
            ids[i, :n] = torch.tensor(ctx + choices[k])
            mask[i, :n] = 1
        out = model.score(ids.to(dev), attention_mask=mask.to(dev), fp8_weights=fp8_weights)
        lp, gr = out.logprobs.cpu(), out.greedy.cpu()
        for i, (n, q, k) in enumerate(batch):
            c0 = len(requests[q][0])
            total[(q, k)] = (float(lp[i, c0:n].double().sum()), bool(gr[i, c0:n].all()))
    acc = acc_norm = greedy = 0
    for q, (_, choices, gold) in enumerate(requests):
        sums = [total[(q, k)][0] for k in range(len(choices))]
        per_tok = [s / len(c) for s, c in zip(sums, choices)]
        acc += max(range(len(sums)), key=lambda k: sums[k]) == gold
        acc_norm += max(range(len(per_tok)), key=lambda k: per_tok[k]) == gold
        greedy += total[(q, gold)][1]
    n = len(requests)
    return {"acc": acc / n, "acc_per_token": acc_norm / n, "greedy": greedy / n, "n": n}


def main(argv=None) -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    add_model_args(ap)
    ap.add_argument("--tokens", default=None, help="glob of token shards (write_token_shard / tokenize_corpus.py) for perplexity")
    ap.add_argument("--seq-len", type=int, default=1024)
    ap.add_argument("--batch-size", type=int, default=8, help="sequences per score() call")
    ap.add_argument("--batches", type=int, default=10, help="perplexity: number of batches to score")
    ap.add_argument("--seed", type=int, default=0, help="perplexity: seed of the window order")
    ap.add_argument("--choices", default=None, help="JSONL file of multiple-choice requests")
    ap.add_argument("--tokenizer", default=None, help="local tokenizer directory for text requests (never downloaded)")
    ap.add_argument("--fp8-weights", action="store_true",
                    help="score the model with its decoder-layer projections quantised to e4m3 (generate --fp8-weights): "
                         "compare with a run without it to see what the quantisation costs")
    a = ap.parse_args(argv)
    if a.tokens is None and a.choices is None:
        ap.error("give --tokens (perplexity) and/or --choices (multiple choice)")
    if a.batch_size < 1 or a.batches < 1 or a.seq_len < 2:
        ap.error("--batch-size and --batches must be >= 1, --seq-len >= 2")
    tok = None
    if a.tokenizer is not None:
        from transformers import AutoTokenizer

        tok = AutoTokenizer.from_pretrained(a.tokenizer, local_files_only=True)
    model = load_model(a)
    result = {}
    if a.tokens is not None:
        result.update(perplexity(model, a.tokens, a.seq_len, a.batch_size, a.batches, a.seed, a.fp8_weights))
    if a.choices is not None:
        result.update(multiple_choice(model, a.choices, a.batch_size, tok, a.fp8_weights))
    if a.fp8_weights:
        result["fp8_weights"] = True
    print(json.dumps(result))


if __name__ == "__main__":
    main()
