#!/usr/bin/env python
"""Generate text with a Llama model: an HF directory, a preset (random weights from --init-seed), or a training checkpoint.

    python scripts/generate.py --model 150m --checkpoint outputs/model_step_1000 --weights outer --prompt-ids "1 450 4996"
    python scripts/generate.py --model /models/llama-150m --prompt "The capital of" --tokenizer /models/llama-150m \\
        --max-new-tokens 64 --do-sample --temperature 0.8 --top-p 0.95
    python scripts/generate.py --model 1b --checkpoint outputs_1b/model_step_1000 --assistant-model 150m \\
        --assistant-checkpoint outputs_150m/model_step_1000 --num-assistant-tokens 4 --prompt-ids "1 450 4996"
    python scripts/generate.py --model 1b --checkpoint outputs_1b/model_step_1000 --num-beams 4 --num-return-sequences 2 \\
        --prompt-ids "1 450 4996"
    python scripts/generate.py --model 150m --checkpoint outputs/model_step_1000 --weights outer --num-beams 4 \\
        --no-repeat-ngram-size 3 --repetition-penalty 1.2 --prompt-ids "1 450 4996"

``--checkpoint`` reads a checkpoint directory written by train_fsdp / utils/ckpt.save_checkpoint (the one holding the
``*.distcp`` shards, i.e. ``model_step_N`` or its ``diloco_rank_R`` sub-directory).  ``--weights local`` takes the
worker's own weights (``model``), ``--weights outer`` the DiLoCo global model (``theta_outer``).  Tokenizers are only
read from a local directory.  ``--assistant-model`` (with ``--assistant-checkpoint`` / ``--assistant-weights``) loads a
draft model the same way and turns on assisted (speculative) generation.  ``--num-beams`` > 1 runs beam search and prints
each returned hypothesis with its score (``--num-return-sequences`` per prompt).  ``--repetition-penalty``,
``--no-repeat-ngram-size`` and ``--min-new-tokens`` are HF's repetition controls, for greedy, sampling and beam search.
``--prompt-lookup-num-tokens`` (with ``--max-matching-ngram-size``) turns on prompt lookup decoding: speculative
generation whose proposals are copied from the row's own prompt and output, with no draft model.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from opendiloco_b200.models.config import LlamaConfig  # noqa: E402
from opendiloco_b200.models.llama import LlamaForCausalLM  # noqa: E402


def load_checkpoint_weights(model: LlamaForCausalLM, ckpt_dir: str, weights: str) -> None:
    """Copy the flat ``model`` (local) or ``theta_outer`` (outer) range of a checkpoint into the model's master weights."""
    from opendiloco_b200.utils import ckpt

    meta_path = os.path.join(ckpt_dir, ckpt.METADATA_FILE)
    if not os.path.isfile(meta_path):
        raise SystemExit(f"error: {ckpt_dir} has no {ckpt.METADATA_FILE}: not a flat-arena checkpoint directory")
    with open(meta_path) as f:
        meta = json.load(f)
    numel = int(meta["numel"])
    if numel != model.arena.numel:
        raise SystemExit(f"error: checkpoint holds {numel} parameters, model --model has {model.arena.numel}: wrong --model?")
    key = {"local": "model", "outer": "theta_outer"}[weights]
    ckpt._SHARD_CACHE.clear()
    try:
        flat = ckpt._assemble(ckpt_dir, key, 0, numel, "cpu")
    finally:
        ckpt._SHARD_CACHE.clear()
    if flat is None:
        raise SystemExit(f"error: checkpoint {ckpt_dir} has no '{key}' weights"
                         + (" (it was written without a DiLoCo optimizer, so there is no outer model)" if weights == "outer" else ""))
    with torch.no_grad():
        model.arena.master.copy_(flat.to(model.arena.device))
    model.arena.sync_shadow()


def parse_bad_words(text: str | None) -> list[list[int]] | None:
    """"12 13;99" -> [[12, 13], [99]]."""
    if text is None:
        return None
    return [[int(t) for t in seq.split()] for seq in text.split(";") if seq.strip()]


def parse_sequence_bias(text: str | None) -> dict[tuple[int, ...], float] | None:
    """"12 13:-2.5;99:1.0" -> {(12, 13): -2.5, (99,): 1.0}."""
    if text is None:
        return None
    out = {}
    for item in text.split(";"):
        if not item.strip():
            continue
        ids, _, bias = item.rpartition(":")
        out[tuple(int(t) for t in ids.split())] = float(bias)
    return out


def add_model_args(ap: argparse.ArgumentParser) -> None:
    """The options that choose the model and its weights (shared with scripts/evaluate.py)."""
    ap.add_argument("--model", required=True, help="HF model directory or preset name (150m, 1b, ...)")
    ap.add_argument("--checkpoint", default=None, help="training checkpoint directory to take the weights from")
    ap.add_argument("--weights", choices=["local", "outer"], default="local", help="with --checkpoint: local or DiLoCo outer weights")
    ap.add_argument("--init-seed", type=int, default=0, help="seed of the random weights of a preset without weights")
    ap.add_argument("--device", default="cuda" if torch.cuda.is_available() else "cpu")
    ap.add_argument("--precision", default=None, help="bf16-mixed (default on CUDA), 32-true (default on CPU), fp16-mixed")


def load_model(a: argparse.Namespace, model: str | None = None, checkpoint: str | None = None,
               weights: str | None = None) -> LlamaForCausalLM:
    """The model chosen by the ``add_model_args`` options, or by the given model / checkpoint / weights, in eval mode."""
    if model is None:
        model, checkpoint, weights = a.model, a.checkpoint, a.weights
    device = torch.device(a.device)
    precision = a.precision or ("bf16-mixed" if device.type == "cuda" else "32-true")
    cfg = LlamaConfig.from_pretrained(model)
    if checkpoint is not None:
        m = LlamaForCausalLM(cfg, device=device, precision=precision, init=False)
        load_checkpoint_weights(m, checkpoint, weights)
    else:
        m = LlamaForCausalLM.from_pretrained(model, config=cfg, device=device, precision=precision, seed=a.init_seed)
    return m.eval()


def main(argv=None) -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    add_model_args(ap)
    ap.add_argument("--prompt-ids", action="append", default=None, help='space-separated token ids; repeat for a batch')
    ap.add_argument("--prompt", action="append", default=None, help="prompt text (needs --tokenizer); repeat for a batch")
    ap.add_argument("--tokenizer", default=None, help="local tokenizer directory (never downloaded)")
    ap.add_argument("--max-new-tokens", type=int, default=20)
    ap.add_argument("--do-sample", action="store_true")
    ap.add_argument("--temperature", type=float, default=1.0)
    ap.add_argument("--top-k", type=int, default=50)
    ap.add_argument("--top-p", type=float, default=1.0)
    ap.add_argument("--eos-token-id", type=int, default=None)
    ap.add_argument("--pad-token-id", type=int, default=None)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--assistant-model", default=None, help="draft model (HF directory or preset) for assisted generation")
    ap.add_argument("--assistant-checkpoint", default=None, help="training checkpoint directory of the draft's weights")
    ap.add_argument("--assistant-weights", choices=["local", "outer"], default="local",
                    help="with --assistant-checkpoint: local or DiLoCo outer weights")
    ap.add_argument("--num-assistant-tokens", type=int, default=4, help="draft tokens proposed per round (1..7)")
    ap.add_argument("--num-beams", type=int, default=1, help="beam search with this many beams (1..8); 1: greedy / sampling")
    ap.add_argument("--length-penalty", type=float, default=1.0, help="beam search: hypothesis score = sum log p / length ** this")
    ap.add_argument("--early-stopping", choices=["true", "false", "never"], default="false",
                    help="beam search: HF's early_stopping (true, false or never)")
    ap.add_argument("--num-return-sequences", type=int, default=1,
                    help="beam search: hypotheses returned per prompt; with --do-sample: independent samples per prompt")
    ap.add_argument("--repetition-penalty", type=float, default=1.0, help="HF's repetition penalty on the row's history (1.0: off)")
    ap.add_argument("--no-repeat-ngram-size", type=int, default=0, help="no n-gram of this size occurs twice in a row (0: off)")
    ap.add_argument("--min-new-tokens", type=int, default=0, help="EOS is forbidden until this many new tokens (0: off)")
    ap.add_argument("--prompt-lookup-num-tokens", type=int, default=None,
                    help="prompt lookup decoding: tokens proposed per round from the row's own history (1..7)")
    ap.add_argument("--max-matching-ngram-size", type=int, default=None, help="prompt lookup: longest n-gram matched (default 2)")
    ap.add_argument("--fp8-weights", action="store_true",
                    help="quantise the decoder-layer projections to e4m3 (one scale per output row) and decode on them")
    ap.add_argument("--fp8-kv-cache", action="store_true",
                    help="keep the KV cache in e4m3 with one power-of-two scale per (position, kv head) row")
    ap.add_argument("--bad-words-ids", default=None, help='sequences that must not be generated, e.g. "12 13;99"')
    ap.add_argument("--sequence-bias", default=None, help='bias of the last id of each sequence, e.g. "12 13:-2.5;99:1.0"')
    ap.add_argument("--min-length", type=int, default=0, help="EOS is forbidden while prompt + new tokens are shorter (0: off)")
    ap.add_argument("--min-p", type=float, default=None, help="sampling: keep tokens with p >= min_p * p_max (off by default)")
    ap.add_argument("--print-logprobs", action="store_true",
                    help="print each generated token with its log-probability (compute_transition_scores, normalize_logits=True)")
    a = ap.parse_args(argv)
    if a.assistant_model is None and a.assistant_checkpoint is not None:
        ap.error("--assistant-checkpoint needs --assistant-model")

    tok = None
    if a.tokenizer is not None:
        from transformers import AutoTokenizer

        tok = AutoTokenizer.from_pretrained(a.tokenizer, local_files_only=True)
    if (a.prompt is None) == (a.prompt_ids is None):
        ap.error("give exactly one of --prompt-ids or --prompt")
    if a.prompt is not None and tok is None:
        ap.error("--prompt needs --tokenizer")
    prompts = ([[int(t) for t in p.split()] for p in a.prompt_ids] if a.prompt_ids is not None
               else [tok(p)["input_ids"] for p in a.prompt])
    if any(len(p) == 0 for p in prompts):
        ap.error("empty prompt")

    device = torch.device(a.device)
    model = load_model(a)
    assistant = None
    if a.assistant_model is not None:
        assistant = load_model(a, a.assistant_model, a.assistant_checkpoint, a.assistant_weights)

    # left-pad the batch to a common length
    P = max(len(p) for p in prompts)
    ids = torch.zeros(len(prompts), P, dtype=torch.int64)
    mask = torch.zeros(len(prompts), P, dtype=torch.int64)
    for i, p in enumerate(prompts):
        ids[i, P - len(p):] = torch.tensor(p)
        mask[i, P - len(p):] = 1
    early_stopping = {"true": True, "false": False, "never": "never"}[a.early_stopping]
    res = model.generate(ids.to(device), attention_mask=mask.to(device), max_new_tokens=a.max_new_tokens, do_sample=a.do_sample,
                         temperature=a.temperature, top_k=a.top_k, top_p=a.top_p, eos_token_id=a.eos_token_id,
                         pad_token_id=a.pad_token_id, seed=a.seed, assistant_model=assistant,
                         num_assistant_tokens=a.num_assistant_tokens, num_beams=a.num_beams, length_penalty=a.length_penalty,
                         early_stopping=early_stopping, num_return_sequences=a.num_return_sequences, return_dict_in_generate=True,
                         repetition_penalty=a.repetition_penalty, no_repeat_ngram_size=a.no_repeat_ngram_size,
                         min_new_tokens=a.min_new_tokens, prompt_lookup_num_tokens=a.prompt_lookup_num_tokens,
                         max_matching_ngram_size=a.max_matching_ngram_size, fp8_weights=a.fp8_weights,
                         fp8_kv_cache=a.fp8_kv_cache, bad_words_ids=parse_bad_words(a.bad_words_ids),
                         sequence_bias=parse_sequence_bias(a.sequence_bias), min_length=a.min_length, min_p=a.min_p,
                         output_scores=a.print_logprobs)
    out = res.sequences.cpu()
    logprobs = (model.compute_transition_scores(res.sequences, res.scores, res.beam_indices, normalize_logits=True).cpu()
                if a.print_logprobs else None)
    R = out.shape[0] // len(prompts)
    for i, p in enumerate(prompts):
        for r in range(R):
            new = out[i * R + r, P:].tolist()
            if res.sequences_scores is not None:
                print(f"score: {float(res.sequences_scores[i * R + r]):.6f}")
            print("ids:", " ".join(str(t) for t in p + new))
            if logprobs is not None:                 # beam search: the hypothesis' own tokens, EOS included
                n = int((res.beam_indices[i * R + r] >= 0).sum()) if res.beam_indices is not None else len(new)
                print("logprobs:", " ".join(f"{t}:{float(lp):.4f}" for t, lp in zip(new[:n], logprobs[i * R + r, :n].tolist())))
            if tok is not None:
                print("text:", tok.decode(p + new, skip_special_tokens=True))
    if assistant is not None:
        st = model.engine.assisted_state
        print(f"assisted: {st.verify_passes()} verify passes, acceptance {st.acceptance_rate():.3f}")
    if a.prompt_lookup_num_tokens is not None:
        st = model.engine.assisted_state
        print(f"prompt lookup: {st.verify_passes()} verify passes, acceptance {st.acceptance_rate():.3f}")


if __name__ == "__main__":
    main()
