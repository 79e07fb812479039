"""Host-side mirror of stable_whisper/decode.py for the H100 path: KV-cached decoding of a BATCH of windows -- greedy at
temperature 0, ``best_of`` draws at temperature > 0, the temperature fallback of ``transcribe_stable`` over batch subsets,
per-window prompts (ragged initial tokens).

``decode_stable`` keeps the reference's call shape for one window; ``decode_windows`` is the batched engine:
    encoder output (cached, as DecodingTaskStable._get_audio_features) -> cross K/V ->
    per step: [fused logit filters + pick / draw] -> [decoder step for B sequences]     (decode.py:33-65)
The two kernels-sequences of a step are captured ONCE into a CUDA graph and replayed; every position-dependent value
lives in device memory (position counter, per-sequence sampling state, token/argmax tables indexed by step), so the
host only polls the `done` flags every few steps instead of the reference's per-step ``.all()`` sync.
"""
import zlib
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Union

import numpy as np
import torch

from . import _lib as L
from .model import B200Whisper

CHUNK_LENGTH = 30


@dataclass
class DecodingOptions:              # whisper.decoding.DecodingOptions
    task: str = "transcribe"
    language: Optional[str] = None
    temperature: float = 0.0
    sample_len: Optional[int] = None
    best_of: Optional[int] = None           # independent samples per window at temperature > 0
    beam_size: Optional[int] = None         # beam search: not on the configured path (raises)
    patience: Optional[float] = None
    length_penalty: Optional[float] = None  # MaximumLikelihoodRanker: None = plain length normalisation
    prompt: Optional[Union[str, List[int]]] = None      # previous context, shared by the batch (per window: ``prompts=``)
    prefix: Optional[Union[str, List[int]]] = None      # prefix of the current context
    suppress_tokens: Optional[str] = "-1"
    suppress_blank: bool = True
    without_timestamps: bool = False
    max_initial_timestamp: Optional[float] = 1.0
    fp16: bool = False


@dataclass
class DecodingResult:               # whisper.decoding.DecodingResult
    audio_features: Optional[torch.Tensor]
    language: str
    language_probs: Optional[Dict[str, float]] = None
    tokens: List[int] = field(default_factory=list)
    text: str = ""
    avg_logprob: float = np.nan
    no_speech_prob: float = np.nan
    temperature: float = np.nan
    compression_ratio: float = np.nan


def compression_ratio(text: str) -> float:
    b = text.encode("utf-8")
    return len(b) / len(zlib.compress(b))


def _suppress_list(tokenizer, options: DecodingOptions) -> List[int]:
    st = options.suppress_tokens
    if isinstance(st, str):
        st = [int(t) for t in st.split(",")]
    st = list(st or [])
    if -1 in st:
        st = [t for t in st if t >= 0] + list(tokenizer.non_speech_tokens)
    st += [tokenizer.transcribe, tokenizer.translate, tokenizer.sot, tokenizer.sot_prev, tokenizer.sot_lm]
    if tokenizer.no_speech is not None:
        st.append(tokenizer.no_speech)
    return sorted(set(st))


class StepEngine:
    """Device state of a batch of B decoding sequences + the two launch sequences of one step."""

    def __init__(self, model: B200Whisper, B: int, table_rows: int, reuse_buffers: bool = False,
                 seq_off: Optional[torch.Tensor] = None, cache_rows: Optional[int] = None):
        self.m, self.B, self.rows = model, B, table_rows
        dev, lib, V = model.device, model._lib, model.dims.n_vocab
        self.ldv = (V + 7) // 8 * 8
        # ragged initial tokens: per-sequence first cache row (int32 [B], device) and the rows per sequence of the caches
        self.seq_off = seq_off
        self.cache_rows = int(cache_rows or model.dims.n_text_ctx)
        state_bytes = lib.stb_decode_state_bytes_rows(model._h, B, self.cache_rows)
        if reuse_buffers:      # model-owned: the self-attention K/V cache (rows beyond `pos` are never read) and the workspace
            self.state = model._buf("decode_state", state_bytes)
            self.ws = model._buf("decode_ws", lib.stb_decode_ws_bytes(model._h, B))
            self.ws.zero_()                                                                          # tickets start at 0
        else:
            self.state = torch.zeros(state_bytes, dtype=torch.uint8, device=dev)
            self.ws = torch.zeros(lib.stb_decode_ws_bytes(model._h, B), dtype=torch.uint8, device=dev)   # tickets start at 0
        self.pos = torch.zeros(1, dtype=torch.int32, device=dev)
        self.logits = torch.empty(B, self.ldv, dtype=torch.float32, device=dev)
        self.seq = torch.zeros(B, 6, dtype=torch.int32, device=dev)          # stb_seq_state[B]
        self.next = torch.zeros(B, dtype=torch.int32, device=dev)
        self.tok_table = torch.zeros(table_rows, B, dtype=torch.int32, device=dev)
        self.arg_table = torch.zeros(table_rows, B, dtype=torch.int32, device=dev)
        self.forced = None
        self.temperature = 0.0        # > 0: inverse-CDF draws from `uniform` [table_rows, B] (stb_sample)
        self.uniform = None
        self.cap = None               # int32 [B]: per-sequence bound on the number of sampled tokens
        self.graph = None
        self.graph_nodes = 0          # kernels in the captured step graph

    def reset(self):
        self.pos.zero_()
        self.seq.zero_()
        self.seq[:, 3] = -1                                                   # last_ts = -1

    def feed(self, tokens: torch.Tensor, ckv: torch.Tensor):
        """decoder step for tokens [B] int32 (device) -> self.logits; pos += 1"""
        m = self.m
        L.check(m._lib.stb_decode_step_ragged(m._h, L.ptr(tokens), self.B, L.ptr(self.pos), L.ptr(self.seq_off),
                                              self.cache_rows, L.ptr(ckv), L.ptr(self.state), L.ptr(self.logits), self.ldv,
                                              L.ptr(self.ws), self.ws.numel(), L.stream_ptr()))

    def step(self, ckv, *sample_args):
        """one decoding step: pick the next token from the current logits, then run the decoder on it"""
        self.sample(*sample_args)
        self.feed(self.next, ckv)

    def sample(self, tk, suppress, first_mask, ts_mask, max_initial_ts, apply_ts_rules):
        m = self.m
        L.check(m._lib.stb_sample(L.ptr(self.logits), self.ldv, self.B, m.dims.n_vocab, int(tk.eot),
                                  int(tk.timestamp_begin), int(tk.no_timestamps), L.ptr(suppress), L.ptr(first_mask),
                                  L.ptr(ts_mask), 0 if ts_mask is None or ts_mask.ndim == 1 else int(ts_mask.stride(0)),
                                  int(max_initial_ts), int(apply_ts_rules), L.ptr(self.forced),
                                  L.ptr(self.seq), L.ptr(self.next), L.ptr(self.tok_table), L.ptr(self.arg_table),
                                  self.rows, float(self.temperature), L.ptr(self.uniform), L.ptr(self.cap), L.stream_ptr()))


def enc_select(enc: dict, idx: Sequence[int]) -> dict:
    """Rows ``idx`` (repeats allowed) of an encoder-output dict of ``model.encode``."""
    B = enc["B"]
    sel = torch.as_tensor(list(idx), dtype=torch.long, device=enc["f32"].device)
    d = enc["f32"].shape[-1]
    pick = lambda t: None if t is None else t.view(B, -1, d).index_select(0, sel).reshape(-1, d).contiguous()
    return {"f32": enc["f32"].index_select(0, sel).contiguous(), "hi": pick(enc["hi"]), "lo": pick(enc["lo"]), "B": len(sel)}


def _as_tokens(tokenizer, v) -> List[int]:
    if v is None:
        return []
    return tokenizer.encode(" " + v.strip()) if isinstance(v, str) else [int(t) for t in v]


def initial_tokens(tokenizer, options: DecodingOptions, n_ctx: int, sample_len: int, prompt=None) -> (List[int], int):
    """whisper DecodingTask._get_initial_tokens: [sot_prev, *prompt[-(n_ctx//2-1):]] + sot_sequence + prefix.
    -> (tokens, length of the tail that starts at the SOT token)."""
    tail = list(tokenizer.sot_sequence_including_notimestamps if options.without_timestamps else tokenizer.sot_sequence)
    if options.prefix:
        ptoks = _as_tokens(tokenizer, options.prefix)
        tail = tail + ptoks[-(n_ctx // 2 - sample_len):]          # (-0 keeps the whole prefix, as the reference's slice does)
    ptoks = _as_tokens(tokenizer, prompt if prompt is not None else options.prompt)
    head = [int(tokenizer.sot_prev)] + ptoks[-(n_ctx // 2 - 1):] if ptoks else []
    return head + tail, len(tail)


def decode_windows(model: B200Whisper, *args, **kwargs):
    """See ``_decode_windows``; runs with the model's device current (launches go to that device's current stream)."""
    with L.device_ctx(model.device):
        return _decode_windows(model, *args, **kwargs)


@torch.no_grad()
def _decode_windows(model: B200Whisper, tokenizer, enc: dict, options: Optional[DecodingOptions] = None, *,
                   ts_token_mask: Optional[torch.Tensor] = None, forced_tokens: Optional[torch.Tensor] = None,
                   use_graph: bool = True, poll_every: int = 16, return_step_logits: bool = False, ckv=None,
                   reuse_buffers: bool = False, prompts: Optional[Sequence[Optional[Sequence[int]]]] = None,
                   generator: Optional[torch.Generator] = None, uniform: Optional[torch.Tensor] = None):
    """KV-cached decode of the B windows whose encoder output is ``enc`` (from ``model.encode``): greedy at temperature 0,
    ``best_of`` independent draws per window at temperature > 0 (whisper GreedyDecoder + MaximumLikelihoodRanker).

    ts_token_mask: silent-timestamp suppression (decode.py:14-16): bool [1501] shared by the batch, bool [B, 1501] with one
                   row per window (what the reference computes, original_whisper.py:504-511), a list of B optional [1501]
                   masks (None = nothing suppressed for that window), or None.
    forced_tokens: int [steps, B] -- the token appended at each step instead of the pick (fixed-length scripts for
                   random-weight benchmarks); the argmax of every step is still returned.
    prompts:       per-window previous-context tokens (``decode_options["prompt"] = all_tokens[prompt_reset_since:]``,
                   original_whisper.py:533); ``options.prompt`` is the same prompt for every window.  Windows whose
                   initial tokens differ in length are right-aligned on the step counter (stb_decode_step_ragged).
    generator / uniform: the random stream of temperature > 0: ``uniform`` fp32 [steps, B * best_of] in [0, 1) (or a callable
                   (steps, sequences) -> such a tensor), else ``torch.rand`` under ``generator`` (default generator of the
                   device when None).
    reuse_buffers: keep the cross K/V block, the KV cache and the step workspace in model-owned buffers (the returned
                   ``extras["ckv"]`` is then only valid until the next such call).
    -> (list of DecodingResult, extras dict(step_argmax [steps,B], step_tokens, sum_logprob, ckv))
    """
    options = options or DecodingOptions()
    if options.beam_size is not None:
        raise NotImplementedError("H100 decode path: beam search is not implemented (greedy / sampling only)")
    if options.temperature == 0 and options.best_of is not None:
        raise ValueError("best_of with greedy sampling (T=0) is not compatible")            # DecodingTask._verify_options
    if options.patience is not None:
        raise ValueError("patience requires beam_size to be given")
    if options.length_penalty is not None and not (0 <= options.length_penalty <= 1):
        raise ValueError("length_penalty (alpha) should be a value between 0 and 1")
    temperature = float(options.temperature or 0.0)
    n_group = int(options.best_of or 1) if temperature > 0 else 1
    dev, n_win, V = model.device, enc["B"], model.dims.n_vocab
    n_ctx = model.dims.n_text_ctx
    sample_len = options.sample_len or n_ctx // 2
    if prompts is not None and len(prompts) != n_win:
        raise ValueError(f"prompts: {len(prompts)} entries for {n_win} windows")
    inits, tails = zip(*[initial_tokens(tokenizer, options, n_ctx, sample_len, None if prompts is None else prompts[w])
                         for w in range(n_win)])
    tail_len = tails[0]
    if n_group > 1:                                        # tokens.repeat_interleave(n_group) (DecodingTask.run)
        if ckv is not None:
            raise ValueError("best_of > 1: pass `enc`, not a precomputed cross K/V block")
        rep = [w for w in range(n_win) for _ in range(n_group)]
        enc = enc_select(enc, rep)
        inits = [inits[w] for w in rep]
    B = enc["B"]
    lens = [len(t) for t in inits]
    max_init, min_init = max(lens), min(lens)
    ragged = max_init != min_init
    steps = sample_len if forced_tokens is None else min(sample_len, int(forced_tokens.shape[0]))
    # a sequence stops once `tokens.shape[-1] > n_ctx` (decode.py:60): at most n_ctx - len(initial) + 1 sampled tokens
    caps = [n_ctx - n + 1 for n in lens]
    steps = max(min(steps, max(caps)), 0)
    seq_off = torch.tensor([max_init - n for n in lens], dtype=torch.int32, device=dev) if ragged else None
    # (tests/standin.py swaps the engine for a CPU one built on the oracle to pin this host logic without a GPU)
    engine_cls = getattr(model, "step_engine_cls", None) or StepEngine
    eng = engine_cls(model, B, max(steps, 1), reuse_buffers=reuse_buffers, seq_off=seq_off,
                     cache_rows=n_ctx + (max_init - min_init))
    eng.reset()
    if min(caps) < steps:
        eng.cap = torch.tensor(caps, dtype=torch.int32, device=dev)
    if temperature > 0:
        eng.temperature = temperature
        if callable(uniform):
            uniform = uniform(max(steps, 1), B)
        if uniform is None:
            gdev = generator.device if generator is not None else dev
            uniform = torch.rand(max(steps, 1), B, generator=generator, device=gdev)
        if tuple(uniform.shape) != (max(steps, 1), B):
            raise ValueError(f"uniform: expected shape {(max(steps, 1), B)}, got {tuple(uniform.shape)}")
        eng.uniform = uniform.to(dev, torch.float32).contiguous()
    if ckv is None:
        ckv = model.cross_kv(enc, decode=True, reuse=reuse_buffers)
    # filter tables (SuppressTokens, SuppressBlank)
    sup = torch.zeros(V, dtype=torch.uint8)
    sup[_suppress_list(tokenizer, options)] = 1 if options.suppress_tokens else 0
    first = torch.zeros(V, dtype=torch.uint8)
    if options.suppress_blank:
        first[tokenizer.encode(" ") + [tokenizer.eot]] = 1
    sup, first = sup.to(dev), first.to(dev)
    tsm = None
    if ts_token_mask is not None:
        if isinstance(ts_token_mask, (list, tuple)):
            if len(ts_token_mask) != n_win:
                raise ValueError(f"ts_token_mask: {len(ts_token_mask)} masks for {n_win} windows")
            rows = torch.zeros(n_win, 1501, dtype=torch.uint8)
            for i, mk in enumerate(ts_token_mask):
                if mk is not None:
                    rows[i] = torch.as_tensor(mk).to(torch.uint8)
            ts_token_mask = rows
        if ts_token_mask.ndim == 2 and ts_token_mask.shape[0] != n_win:
            raise ValueError(f"ts_token_mask: {ts_token_mask.shape[0]} rows for {n_win} windows")
        if ts_token_mask.shape[-1] != 1501:
            raise ValueError("ts_token_mask must have 1501 entries per window")
        if ts_token_mask.ndim == 2 and n_group > 1:
            ts_token_mask = ts_token_mask.repeat_interleave(n_group, dim=0)
        tsm = ts_token_mask.to(torch.uint8).to(dev).contiguous()
    apply_rules = not options.without_timestamps
    max_init_ts = -1
    if apply_rules and options.max_initial_timestamp:
        max_init_ts = round(options.max_initial_timestamp / (CHUNK_LENGTH / model.dims.n_audio_ctx))
    if forced_tokens is not None:
        eng.forced = forced_tokens[:steps].to(dev, torch.int32).contiguous()
    # ---- initial tokens: one step each, right-aligned (every sequence's SOT token is fed at the same step); the logits at
    # the SOT position give no_speech_prob (decode.py:42-44)
    init_table = torch.full((max_init, B), int(tokenizer.eot), dtype=torch.int32)
    for b, t in enumerate(inits):
        init_table[max_init - len(t):, b] = torch.tensor(t, dtype=torch.int32)
    init_table = init_table.to(dev)
    no_speech = [float("nan")] * B
    sot_step = max_init - tail_len + list(inits[0][-tail_len:]).index(tokenizer.sot)
    for i in range(max_init):
        eng.feed(init_table[i], ckv)
        if i == sot_step and tokenizer.no_speech is not None:
            p, _ = model.token_probs(eng.logits, V, torch.full((B,), int(tokenizer.no_speech)))
            no_speech = p.cpu().tolist()
    step_logits = []

    def one_step():
        eng.step(ckv, tokenizer, sup, first, tsm, max_init_ts, apply_rules)

    done_steps = 0
    # step 0 runs eagerly (also warms every kernel), the rest replay a captured graph; the LAST step only samples -- the
    # decoder forward of its token would produce logits nobody reads (and, at the n_ctx stop, a position past the table)
    on_cuda = torch.device(dev).type == "cuda"
    if return_step_logits or not on_cuda:
        use_graph = False
    while done_steps < steps:
        if done_steps == steps - 1:
            eng.sample(tokenizer, sup, first, tsm, max_init_ts, apply_rules)
            if return_step_logits:
                step_logits.append(eng.logits[:, :V].clone())
        elif return_step_logits:
            eng.sample(tokenizer, sup, first, tsm, max_init_ts, apply_rules)
            step_logits.append(eng.logits[:, :V].clone())
            eng.feed(eng.next, ckv)
        elif use_graph and done_steps >= 1:
            if eng.graph is None:
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                c0 = model._lib.stb_launch_count()
                with torch.cuda.graph(g):
                    one_step()                          # this capture pass does not execute; replay below does
                eng.graph = g
                eng.graph_nodes = int(model._lib.stb_launch_count() - c0)
                model.graph_kernel_launches -= eng.graph_nodes      # counted by the library at capture, but not executed
            eng.graph.replay()
            model.graph_kernel_launches += eng.graph_nodes          # kernels executed by this replay
        else:
            one_step()
        done_steps += 1
        if forced_tokens is None and done_steps % poll_every == 0 and done_steps < steps:
            if bool((eng.seq[:, 4] != 0).all()):        # every sequence has emitted EOT
                break
    if on_cuda:
        torch.cuda.synchronize()
    toks = eng.tok_table[:done_steps].cpu().numpy()
    args = eng.arg_table[:done_steps].cpu().numpy()
    sum_lp = eng.seq[:, 5].contiguous().view(torch.float32).cpu().numpy()
    seqs = []
    for b in range(B):
        seq = toks[:, b].tolist()[: caps[b]]
        if tokenizer.eot in seq:
            seq = seq[: seq.index(tokenizer.eot)]
        seqs.append(seq)
    results, chosen = [], []
    for w in range(n_win):
        grp = range(w * n_group, (w + 1) * n_group)
        if n_group > 1:                                  # MaximumLikelihoodRanker.rank
            def score(b):
                n = len(seqs[b])
                pen = n if options.length_penalty is None else ((5 + n) / 6) ** options.length_penalty
                return float(sum_lp[b]) / pen if pen else float("-inf")
            b = grp[int(np.argmax([score(b) for b in grp]))]
        else:
            b = grp[0]
        chosen.append(b)
        seq = seqs[b]
        text = tokenizer.decode(seq).strip()
        results.append(DecodingResult(audio_features=enc["f32"][b], language=options.language or "en", tokens=seq, text=text,
                                      avg_logprob=float(sum_lp[b]) / (len(seq) + 1), no_speech_prob=no_speech[b],
                                      temperature=temperature, compression_ratio=compression_ratio(text) if text else float("nan")))
    extras = dict(step_argmax=args, step_tokens=toks, sum_logprob=sum_lp, ckv=ckv, step_logits=step_logits,
                  steps=done_steps, chosen=chosen, n_group=n_group)
    return results, extras


def needs_fallback(result: DecodingResult, compression_ratio_threshold: Optional[float], logprob_threshold: Optional[float],
                   no_speech_threshold: Optional[float]) -> bool:
    """The test of ``decode_with_fallback`` (original_whisper.py:371-389)."""
    need = False
    if compression_ratio_threshold is not None and result.compression_ratio > compression_ratio_threshold:
        need = True                                      # too repetitive
    if logprob_threshold is not None and result.avg_logprob < logprob_threshold:
        need = True                                      # average log probability is too low
    if no_speech_threshold is not None and result.no_speech_prob > no_speech_threshold:
        need = False                                     # silence
    return need


def decode_with_fallback(model: B200Whisper, tokenizer, enc: dict, options: Optional[DecodingOptions] = None, *,
                         temperature: Union[float, Sequence[float]] = 0.0, compression_ratio_threshold: Optional[float] = 2.4,
                         logprob_threshold: Optional[float] = -1.0, no_speech_threshold: Optional[float] = 0.6,
                         ts_token_mask=None, prompts=None, generator: Optional[torch.Generator] = None,
                         uniforms: Optional[Sequence[Optional[torch.Tensor]]] = None, **kw):
    """Temperature fallback (``decode_with_fallback``, original_whisper.py:349-393) over a BATCH of windows: every window is
    decoded at the first temperature; the windows that fail the compression-ratio / log-prob test are decoded again -- only
    those, gathered into a smaller batch over the cached encoder output -- at the next temperature, and so on.  Per window
    this is exactly the reference's loop (its windows are independent given the prompt).
    ``uniforms[i]``: the random stream of the i-th temperature (tests; columns of windows that are not re-decoded are
    skipped), or a callable (temperature index, steps, sequences) -> fp32 [steps, sequences].
    -> (results, extras of the first pass, n_fallbacks [B])"""
    from dataclasses import replace
    options = options or DecodingOptions()
    temps = [temperature] if isinstance(temperature, (int, float)) else list(temperature)
    B = enc["B"]
    results: List[Optional[DecodingResult]] = [None] * B
    n_fb = [0] * B
    pending = list(range(B))
    first_extras = None
    masks = ts_token_mask
    if masks is not None and not isinstance(masks, (list, tuple)):
        masks = torch.as_tensor(masks)
        masks = [masks[b] for b in range(B)] if masks.ndim == 2 else [masks] * B
    for ti, t in enumerate(temps):
        # t > 0 disables beam_size / patience, t == 0 disables best_of (original_whisper.py:357-364)
        opts = replace(options, temperature=float(t), **(dict(beam_size=None, patience=None) if t > 0 else dict(best_of=None)))
        whole = len(pending) == B
        sub_enc = enc if whole else enc_select(enc, pending)
        sub_kw = dict(kw)
        if not whole:
            sub_kw.pop("ckv", None)
            if sub_kw.get("forced_tokens") is not None:
                sub_kw["forced_tokens"] = sub_kw["forced_tokens"][:, pending]
        if callable(uniforms):                           # (temperature index, steps, sequences) -> fp32 [steps, sequences]
            u = (lambda n_steps, n_seq, ti=ti: uniforms(ti, n_steps, n_seq)) if t > 0 else None
        else:
            u = None if uniforms is None or ti >= len(uniforms) else uniforms[ti]
            if u is not None and not whole:
                g = int(opts.best_of or 1) if t > 0 else 1
                u = u[:, [b * g + k for b in pending for k in range(g)]]
        res, extras = decode_windows(model, tokenizer, sub_enc, opts,
                                     ts_token_mask=None if masks is None else [masks[b] for b in pending],
                                     prompts=None if prompts is None else [prompts[b] for b in pending],
                                     generator=generator, uniform=u, **sub_kw)
        if first_extras is None:
            first_extras = extras
        again = []
        for k, b in enumerate(pending):
            results[b] = res[k]
            if ti + 1 < len(temps) and needs_fallback(res[k], compression_ratio_threshold, logprob_threshold, no_speech_threshold):
                again.append(b)
                n_fb[b] += 1
        pending = again
        if not pending:
            break
    return results, first_extras, n_fb


def decode_stable(model: B200Whisper, mel: torch.Tensor, options: Optional[DecodingOptions] = None,
                  ts_token_mask: Optional[torch.Tensor] = None, audio_features: Optional[dict] = None, **kwargs):
    """Same contract as stable_whisper/decode.py:70-110: -> (DecodingResult | list, audio_features).
    ``audio_features`` is the dict returned by ``model.encode`` (reused across temperature fallbacks)."""
    from .tokenizer import get_tokenizer
    options = options or DecodingOptions()
    for k, v in kwargs.items():
        setattr(options, k, v)
    single = mel.ndim == 2
    if audio_features is None:
        audio_features = model.encode(mel[None] if single else mel)
    tk = get_tokenizer(model, language=options.language or "en", task=options.task,
                       synthetic=getattr(model, "random_init", True))
    res, _ = decode_windows(model, tk, audio_features, options, ts_token_mask=ts_token_mask)
    return (res[0] if single else res), audio_features
