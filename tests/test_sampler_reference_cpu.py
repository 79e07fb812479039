"""A float64 restatement of one decode step's logit filters and pick, pinned to the oracle's own filter classes (CPU).

``restate`` is the reference that ``tests/test_gpu_sampler_fp64.py`` holds ``stb_sample`` to.  For ONE sequence it takes the raw
logits, the FULL list of tokens sampled so far (the kernel only keeps a compressed state of it), the masks, the rule flags and
a uniform, and follows, in order:

* ``SuppressBlank`` (first step only), ``SuppressTokens``, ``ApplyTimestampRules`` (``oracle/whisper_ref/decoding.py``);
* the silent-timestamp mask (``_suppress_ts``), applied after the timestamp rules;
* ``logits.nan_to_num_(-inf)``: masked (-inf) -> -FLT_MAX, NaN -> -inf, +inf -> FLT_MAX;
* ``GreedyDecoder.update``: the argmax (first index on ties) or, at temperature > 0, the inverse-CDF draw of the caller's
  uniform; the log-prob of the pick; the EOT latch; the per-sequence cap on sampled tokens.

The "timestamps outweigh text" rule is decided in float64 (logsumexp of the timestamp logits against the best text logit; a
row holding a NaN or +inf never suppresses text, since the reference's fp32 ``log_softmax`` of such a row is all NaN).  The
masks and clamps need no arithmetic, so the filtered row is float32 and exact.

The test below runs the oracle classes on a ``[1, n]`` token row built from each history, over the three vocabulary layouts,
and requires the same filtered row bit for bit.  Where the oracle's fp32 ``log_softmax`` decides the text-vs-timestamp rule the
other way, the float64 margin must lie inside the near-tie band ``near_tie_band``.
"""
import numpy as np
import pytest
import torch

FLT_MAX = float(np.finfo(np.float32).max)


def near_tie_band(x: np.ndarray) -> float:
    """|logsumexp(timestamps) - max(text)| below which fp32 rounding may decide the rule either way."""
    fin = x[np.isfinite(x)]
    return 1e-5 * (1.0 + (float(np.abs(fin).max()) if fin.size else 0.0))


def new_state():
    """stb_seq_state as the decode loop resets it: n_sampled, last_tok, prev_tok, last_ts, done, sum_logprob."""
    return dict(n_sampled=0, last_tok=0, prev_tok=0, last_ts=-1, done=0, sum_logprob=0.0)


def state_of(history, eot, ts_begin):
    """The compressed state the kernel holds after appending ``history`` (sum_logprob not included)."""
    st = new_state()
    for t in history:
        st = dict(st, n_sampled=st["n_sampled"] + 1, prev_tok=st["last_tok"], last_tok=int(t),
                  last_ts=int(t) if t >= ts_begin else st["last_ts"], done=int(t == eot))
    return st


def rule_masks(V, history, *, eot, ts_begin, no_timestamps, suppress=None, first_mask=None, apply_ts_rules=True,
               max_initial_ts=-1):
    """bool [V]: the indices SuppressBlank / SuppressTokens / ApplyTimestampRules set to -inf, from the whole history."""
    kill = np.zeros(V, dtype=bool)
    n = len(history)
    if suppress is not None:
        kill |= np.asarray(suppress, dtype=bool)
    if n == 0 and first_mask is not None:
        kill |= np.asarray(first_mask, dtype=bool)
    if apply_ts_rules:
        kill[no_timestamps] = True
        last_was_ts = n >= 1 and history[-1] >= ts_begin
        penult_was_ts = n < 2 or history[-2] >= ts_begin
        if last_was_ts:
            if penult_was_ts:
                kill[ts_begin:] = True
            else:
                kill[:eot] = True
        ts = [t for t in history if t >= ts_begin]
        if ts:
            floor = ts[-1] if (last_was_ts and not penult_was_ts) else ts[-1] + 1
            kill[ts_begin:floor] = True
        if n == 0:
            kill[:ts_begin] = True
            if max_initial_ts >= 0:
                kill[ts_begin + max_initial_ts + 1:] = True
    return kill


def ts_margin(x: np.ndarray, ts_begin: int):
    """float64 logsumexp(x[ts_begin:]) - max(x[:ts_begin]) of the masked fp32 row, or None where the reference's rule cannot
    suppress text (a NaN or +inf in the row makes its log_softmax NaN; no finite timestamp leaves ts_lp = -inf)."""
    x = x.astype(np.float64)
    if np.isnan(x).any() or np.isposinf(x).any():
        return None
    ts, text = x[ts_begin:], x[:ts_begin]
    m = ts.max()
    if m == -np.inf:
        return None
    lse = m + np.log(np.exp(ts - m).sum())
    return lse - text.max()


def restate(logits, history, *, eot, ts_begin, no_timestamps, suppress=None, first_mask=None, ts_mask=None,
            apply_ts_rules=True, max_initial_ts=-1, temperature=0.0, u=None, in_table=True, forced=None, cap=None,
            kill_text=None, state=None):
    """One step of one sequence.  ``logits`` fp32 [V] (raw), ``history`` the tokens sampled so far, ``ts_mask`` bool [>= V -
    ts_begin] or None, ``u`` the uniform of this step, ``in_table`` False for a step past the step tables (no draw, no forced
    token: the argmax is appended), ``forced`` the token appended instead of the pick, ``cap`` the sequence's bound on sampled
    tokens.  ``kill_text`` overrides the float64 decision of the timestamp rule (for rows inside the near-tie band).
    -> dict(filtered fp32 [V], argmax, drawn, token, logprob (float64), margin, band, kill_text, gmax, log_s, state)"""
    V = logits.shape[0]
    x = np.array(logits, dtype=np.float32, copy=True)
    x[rule_masks(V, history, eot=eot, ts_begin=ts_begin, no_timestamps=no_timestamps, suppress=suppress,
                 first_mask=first_mask, apply_ts_rules=apply_ts_rules, max_initial_ts=max_initial_ts)] = -np.inf
    margin = ts_margin(x, ts_begin) if apply_ts_rules else None
    band = near_tie_band(x)
    if kill_text is None:
        kill_text = margin is not None and margin > 0
    if apply_ts_rules and kill_text:
        x[:ts_begin] = -np.inf
    if ts_mask is not None:
        x[ts_begin:][np.asarray(ts_mask, dtype=bool)[: V - ts_begin]] = -np.inf
    x = np.nan_to_num(x, nan=-np.inf, posinf=FLT_MAX, neginf=-FLT_MAX).astype(np.float32)
    xd = x.astype(np.float64)
    gmax = xd.max()
    log_s = float(np.log(np.exp(xd - gmax).sum()))
    arg = int(np.argmax(xd))
    drawn = arg
    if temperature > 0 and in_table:
        c = np.cumsum(np.exp((xd - gmax) / temperature))
        hit = np.nonzero(c > float(u) * c[-1])[0]
        if hit.size:
            drawn = int(hit[0])
    lp = (xd[drawn] - gmax) - log_s
    st = dict(state) if state is not None else dict(state_of(history, eot, ts_begin), sum_logprob=0.0)
    n = len(history)
    was_done = (n >= 1 and history[-1] == eot) or (cap is not None and n >= cap)
    token = int(forced) if (forced is not None and in_table) else drawn
    if was_done:
        token = eot
    else:
        st["sum_logprob"] = st["sum_logprob"] + lp
    st.update(n_sampled=n + 1, prev_tok=st["last_tok"], last_tok=token,
              last_ts=token if token >= ts_begin else st["last_ts"], done=int(token == eot))
    return dict(filtered=x, argmax=arg, drawn=drawn, token=token, logprob=lp, margin=margin, band=band,
                kill_text=bool(apply_ts_rules and kill_text), gmax=gmax, log_s=log_s, was_done=was_done, state=st)


# ---------------------------------------------------------------------------------------------------------------------------
# random rows and histories shared with the GPU test

LAYOUTS = [(False, 99), (True, 99), (True, 100)]          # n_vocab 51864 (English-only), 51865, 51866 (large-v3)


def layout_tokenizer(multilingual, num_languages):
    from stable_ts_b200.tokenizer import get_tokenizer
    tk = get_tokenizer(multilingual=multilingual, num_languages=num_languages, language="en", task="transcribe",
                       synthetic=True)
    return tk, int(tk.timestamp_begin) + 1501


def random_history(rng, eot, ts_begin, V, max_len=24):
    """A history a decode could append: text, timestamps (paired or lone, rising or not) and special tokens, EOT at the end
    only."""
    n = int(rng.integers(0, max_len + 1))
    h = []
    for _ in range(n):
        r = rng.random()
        if r < 0.4:
            h.append(int(rng.integers(ts_begin, V)))
        elif r < 0.43:
            h.append(int(rng.integers(eot + 1, ts_begin)))
        else:
            h.append(int(rng.integers(0, eot)))
    if h and rng.random() < 0.1:
        h[-1] = eot
    return h


def random_row(rng, V, ts_begin, tie_scale=None):
    """fp32 logits whose timestamp block competes with the text (the rule fires about half the time); ``tie_scale`` plants
    the timestamp logsumexp at that margin above / below the best text logit."""
    x = rng.standard_normal(V) * rng.uniform(0.5, 4.0)
    x[ts_begin:] += rng.uniform(-4.0, 4.0) - np.log(V - ts_begin) + 2.0
    if tie_scale is not None:
        ts = x[ts_begin:]
        lse = ts.max() + np.log(np.exp(ts - ts.max()).sum())
        x[ts_begin:] += x[:ts_begin].max() - lse + tie_scale
    return x.astype(np.float32)


def _oracle_step(logits, history, tk, sample_begin, suppress_list, max_initial_ts, ts_mask, apply_ts_rules):
    from oracle.whisper_ref import decoding as D
    prefix = list(tk.sot_sequence)[:sample_begin] + [int(tk.sot)] * (sample_begin - len(tk.sot_sequence))
    tokens = torch.tensor([prefix + list(history)], dtype=torch.long)
    lg = torch.from_numpy(logits.copy())[None]
    filters = [D.SuppressBlank(tk, sample_begin), D.SuppressTokens(suppress_list)]
    if apply_ts_rules:
        filters.append(D.ApplyTimestampRules(tk, sample_begin, None if max_initial_ts < 0 else max_initial_ts))
    for f in filters:
        f.apply(lg, tokens)
    if ts_mask is not None:
        lg[:, tk.timestamp_begin:][:, torch.from_numpy(ts_mask)] = -np.inf
    lg.nan_to_num_(-np.inf)
    sum_lp = torch.zeros(1)
    new_tokens, _ = D.GreedyDecoder(0.0, tk.eot).update(tokens, lg.clone(), sum_lp)
    return lg[0].numpy(), int(new_tokens[0, -1]), float(sum_lp[0])


@pytest.mark.parametrize("layout", LAYOUTS, ids=["51864", "51865", "51866"])
def test_restatement_equals_the_oracle_filters(layout):
    from stable_ts_b200.decode import DecodingOptions, _suppress_list
    tk, V = layout_tokenizer(*layout)
    eot, ts_begin, no_ts = int(tk.eot), int(tk.timestamp_begin), int(tk.no_timestamps)
    sup_list = _suppress_list(tk, DecodingOptions())
    sup = np.zeros(V, dtype=bool)
    sup[sup_list] = True
    first = np.zeros(V, dtype=bool)
    first[tk.encode(" ") + [eot]] = True
    rng = np.random.default_rng(1000 + V)
    n_rows, n_disagree, n_ties, worst_lp = 1200, 0, 0, 0.0
    for r in range(n_rows):
        history = random_history(rng, eot, ts_begin, V)
        planted = r % 8 == 0
        x = random_row(rng, V, ts_begin, tie_scale=float(rng.choice([-1e-7, 1e-7, -1e-3, 1e-3])) if planted else None)
        kind = r % 23
        if kind == 1:
            x[int(rng.integers(0, ts_begin))] = np.nan                     # NaN among the text logits
        elif kind == 2:
            x[int(rng.integers(ts_begin, V))] = np.nan
        elif kind == 3:
            x[no_ts] = np.nan                                               # NaN where a filter writes -inf
        elif kind == 4:
            x[int(rng.integers(0, V))] = np.inf
        elif kind == 5:
            x[:] = -np.inf
        elif kind == 6:
            x[ts_begin:] = -np.inf
        max_init = int(rng.choice([-1, 0, 50]))
        ts_mask = None
        if r % 3 == 0:
            ts_mask = rng.random(1501) < 0.3
        apply_rules = r % 7 != 0
        sample_begin = len(tk.sot_sequence) + int(rng.integers(0, 3))
        got_o, tok_o, lp_o = _oracle_step(x, history, tk, sample_begin, sup_list, max_init, ts_mask, apply_rules)
        ref = restate(x, history, eot=eot, ts_begin=ts_begin, no_timestamps=no_ts, suppress=sup, first_mask=first,
                      ts_mask=ts_mask, apply_ts_rules=apply_rules, max_initial_ts=max_init)
        if not np.array_equal(got_o.view(np.int32), ref["filtered"].view(np.int32)):
            # the only admissible difference: fp32 log_softmax deciding a near tie the other way
            assert ref["margin"] is not None and abs(ref["margin"]) <= ref["band"], (r, history, ref["margin"])
            alt = restate(x, history, eot=eot, ts_begin=ts_begin, no_timestamps=no_ts, suppress=sup, first_mask=first,
                          ts_mask=ts_mask, apply_ts_rules=apply_rules, max_initial_ts=max_init,
                          kill_text=not ref["kill_text"])
            assert np.array_equal(got_o.view(np.int32), alt["filtered"].view(np.int32)), r
            n_disagree += 1
            continue
        if ref["margin"] is not None and abs(ref["margin"]) <= ref["band"]:
            n_ties += 1
        was_done = bool(history) and history[-1] == eot
        assert tok_o == ref["token"], (r, tok_o, ref["token"])
        if not was_done and np.isfinite(lp_o):
            err = abs(lp_o - ref["logprob"])
            worst_lp = max(worst_lp, err)
            assert err <= 2e-6 * (abs(ref["gmax"]) + abs(ref["gmax"] + ref["log_s"]) + 1.0), (r, lp_o, ref["logprob"])
    print(f"V={V}: {n_rows} rows, restatement == oracle filters; {n_ties} near ties agreed, {n_disagree} near-tie "
          f"disagreements (fp32 log_softmax vs float64); worst log-prob |diff| vs the oracle's fp32 {worst_lp:.2e}")


def test_restatement_state_matches_the_history():
    """The compressed state yields the masks of the history it was built from: state_of is the kernel's update rule."""
    tk, V = layout_tokenizer(True, 100)
    eot, ts_begin = int(tk.eot), int(tk.timestamp_begin)
    rng = np.random.default_rng(5)
    for _ in range(300):
        h = random_history(rng, eot, ts_begin, V)
        st = new_state()
        for i, t in enumerate(h):
            x = random_row(rng, V, ts_begin)
            ref = restate(x, h[:i], eot=eot, ts_begin=ts_begin, no_timestamps=int(tk.no_timestamps), forced=t,
                          state=st)
            if ref["was_done"]:
                break
            st = ref["state"]
        else:
            want = state_of(h, eot, ts_begin)
            assert {k: st[k] for k in want if k != "sum_logprob"} == {k: want[k] for k in want if k != "sum_logprob"}
