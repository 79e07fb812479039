"""``stb_sample`` (the decode step's logit filters + pick, ``csrc/decode.cu``) against the float64 restatement of
``tests/test_sampler_reference_cpu.py``, which that file pins to the oracle's own filter classes.

The kernel works from a compressed per-sequence state (``n_sampled``, ``last_tok``, ``prev_tok``, ``last_ts``); the restatement
scans the whole history.  Every launch here goes through the raw C entry point on given logits, so the states, masks and
special values a random-weight model may never produce are all reached:

* every state the compressed form must get right, with the timestamp rules on and off and ``max_initial_ts`` -1 / 0 / 50;
* forced multi-step histories that open and close timestamp pairs, follow a lone timestamp with text, force a timestamp below
  the floor and end with EOT, with fresh logits at every step and the silent-timestamp mask shared / per row at pitch 1501 /
  per row at pitch 1504;
* the "timestamps outweigh text" rule at planted margins of +-1e-3 (decided as in float64) and inside the near-tie band (either
  outcome, but all text or none), all-text / all-timestamp / whole-row -inf;
* NaN among the text logits (the reference's all-NaN ``log_softmax`` suppresses no text), NaN among the timestamps, NaN where
  a mask writes -inf, +inf in either range, exact ties;
* B = 1 / 7 / 300, the three vocabulary layouts and a V below the block size, ``ld > V`` with NaN sentinels in the padding
  columns, which must be neither read nor written;
* temperature 0 / 0.7 / 1.0 draws, the EOT latch, the per-sequence cap, and the step tables.  Contract pinned here: a step at
  ``n_sampled >= table_rows`` writes no table entry, reads no forced token and no uniform, and appends the argmax.

Exact: the filtered logits (bitwise: the kernel only masks and clamps), argmax, tokens, tables, every state field except
``sum_logprob``.  Bounded: ``sum_logprob`` against float64, ``SUM_LP_REL`` * (|gmax| + |lse| + 1) per step, accumulated.
"""
import numpy as np
import pytest
import torch

from test_sampler_reference_cpu import LAYOUTS, layout_tokenizer, random_history, random_row, restate, state_of

pytestmark = pytest.mark.gpu

# fp32 rounding of expf, the block sum, logf and the running fp32 sum: a few units in the last place of |gmax| + |lse| + 1 per
# step, i.e. at most 2e-6 of it.  Measured on an NVIDIA H100 80GB HBM3 at 700 W: worst 1.28e-5 absolute, 0.044 of that
# 2e-6 bound over every row and step of this file; the committed bound is 1.25x the worst, rounded up
SUM_LP_REL = 1.2e-7
SENTINEL = np.array([0x7FC0BEEF], dtype=np.int32).view(np.float32)[0]     # a NaN with a payload, in columns V..ld-1
WORST = {"err": 0.0, "ratio": 0.0}


def _gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _ids(tk):
    return dict(eot=int(tk.eot), ts_begin=int(tk.timestamp_begin), no_timestamps=int(tk.no_timestamps))


def _masks(tk, V):
    from stable_ts_b200.decode import DecodingOptions, _suppress_list
    sup = np.zeros(V, dtype=bool)
    sup[_suppress_list(tk, DecodingOptions())] = True
    first = np.zeros(V, dtype=bool)
    first[tk.encode(" ") + [int(tk.eot)]] = True
    return sup, first


class Sampler:
    """B sequences sampled by ``stb_sample``, with the float64 restatement stepped alongside over the full histories."""

    def __init__(self, ids, V, B, rows, *, pad=8, suppress=None, first=None, ts_mask=None, ts_stride=0, apply=1,
                 max_init=-1, T=0.0, uniform=None, cap=None, forced=None, histories=None):
        from stable_ts_b200 import _lib as L
        self.L, self.lib = L, L.lib()
        self.ids, self.V, self.B, self.rows, self.ld = ids, V, B, rows, V + pad
        self.apply, self.max_init, self.T, self.ts_stride = apply, max_init, T, ts_stride
        self.suppress, self.first, self.uniform, self.cap, self.forced = suppress, first, uniform, cap, forced
        self.ts_mask = ts_mask                              # np bool [1501] (stride 0) or [B, ts_stride]
        dev = lambda a, dt: None if a is None else torch.as_tensor(np.ascontiguousarray(a)).to(dt).cuda()
        self.d_sup, self.d_first = dev(suppress, torch.uint8), dev(first, torch.uint8)
        self.d_tsm = dev(ts_mask, torch.uint8)
        self.d_u, self.d_cap, self.d_forced = dev(uniform, torch.float32), dev(cap, torch.int32), dev(forced, torch.int32)
        self.hist = [list(h) for h in (histories or [[]] * B)]
        self.ref_state = [dict(state_of(h, ids["eot"], ids["ts_begin"]), sum_logprob=0.0) for h in self.hist]
        st = np.zeros((B, 6), dtype=np.int32)
        for b, s in enumerate(self.ref_state):
            st[b, :5] = [s["n_sampled"], s["last_tok"], s["prev_tok"], s["last_ts"], s["done"]]
        self.states = torch.from_numpy(st).cuda()
        self.nxt = torch.zeros(B, dtype=torch.int32, device="cuda")
        # tables with 3 spare rows of sentinels: a step past table_rows must write none of them
        self.tok = torch.full((rows + 3, B), -7, dtype=torch.int32, device="cuda")
        self.arg = torch.full((rows + 3, B), -7, dtype=torch.int32, device="cuda")
        self.bound = np.zeros(B)

    def step(self, x):
        """one launch on fp32 logits x [B, V]; checks every output against the restatement"""
        L, B, V, ids = self.L, self.B, self.V, self.ids
        full = np.full((B, self.ld), SENTINEL, dtype=np.float32)
        full[:, :V] = x
        d = torch.from_numpy(full).cuda()
        L.check(self.lib.stb_sample(L.ptr(d), self.ld, B, V, ids["eot"], ids["ts_begin"], ids["no_timestamps"],
                                    L.ptr(self.d_sup), L.ptr(self.d_first), L.ptr(self.d_tsm), self.ts_stride,
                                    self.max_init, self.apply, L.ptr(self.d_forced), L.ptr(self.states), L.ptr(self.nxt),
                                    L.ptr(self.tok), L.ptr(self.arg), self.rows, float(self.T), L.ptr(self.d_u),
                                    L.ptr(self.d_cap), L.stream_ptr()))
        torch.cuda.synchronize()
        out = d.cpu().numpy()
        st, nxt = self.states.cpu().numpy(), self.nxt.cpu().numpy()
        tok, arg = self.tok.cpu().numpy(), self.arg.cpu().numpy()
        assert np.array_equal(out[:, V:].view(np.int32), full[:, V:].view(np.int32)), "padding columns V..ld-1 touched"
        for b in range(B):
            h, n = self.hist[b], len(self.hist[b])
            in_table = n < self.rows
            if self.ts_mask is None:
                tsm = None
            else:
                tsm = self.ts_mask if self.ts_stride == 0 else self.ts_mask[b]
            kw = dict(ids, suppress=self.suppress, first_mask=self.first, ts_mask=tsm, apply_ts_rules=bool(self.apply),
                      max_initial_ts=self.max_init, temperature=self.T, in_table=in_table,
                      u=None if self.uniform is None or not in_table else self.uniform[n, b],
                      forced=None if self.forced is None or not in_table else int(self.forced[n, b]),
                      cap=None if self.cap is None else int(self.cap[b]), state=self.ref_state[b])
            ref = restate(x[b], h, **kw)
            got = out[b, :V]
            if not np.array_equal(got.view(np.int32), ref["filtered"].view(np.int32)):
                # inside the near-tie band either decision is admissible -- but all text or none of it
                assert ref["margin"] is not None and abs(ref["margin"]) <= ref["band"], \
                    (b, n, "filtered logits differ", np.nonzero(got.view(np.int32) != ref["filtered"].view(np.int32))[0][:8],
                     ref["margin"], ref["kill_text"])
                ref = restate(x[b], h, kill_text=not ref["kill_text"], **kw)
                assert np.array_equal(got.view(np.int32), ref["filtered"].view(np.int32)), (b, n)
            if in_table:
                assert arg[n, b] == ref["argmax"], (b, n, arg[n, b], ref["argmax"])
                assert tok[n, b] == ref["token"], (b, n, tok[n, b], ref["token"])
            assert nxt[b] == ref["token"], (b, n, nxt[b], ref["token"], ref["drawn"])
            rs = ref["state"]
            assert st[b, :5].tolist() == [rs["n_sampled"], rs["last_tok"], rs["prev_tok"], rs["last_ts"], rs["done"]], \
                (b, n, st[b, :5].tolist(), rs)
            if not ref["was_done"]:
                g = 0.0 if ref["gmax"] < -1e38 else ref["gmax"]      # a fully masked row: lp = -log V exactly
                self.bound[b] += SUM_LP_REL * (abs(g) + abs(g + ref["log_s"]) + 1.0)
            err = abs(float(st[b:b + 1, 5].view(np.float32)[0]) - rs["sum_logprob"])
            WORST["err"] = max(WORST["err"], err)
            if self.bound[b] > 0:
                WORST["ratio"] = max(WORST["ratio"], err / self.bound[b])
            assert err <= self.bound[b] + 1e-30, (b, n, err, self.bound[b])
            self.hist[b].append(ref["token"])
            self.ref_state[b] = rs
        for r in range(self.rows, self.rows + 3):
            assert (tok[r] == -7).all() and (arg[r] == -7).all(), "table row past table_rows written"
        return out


def _state_histories(eot, ts_begin, V):
    """Histories covering n_sampled 0 / 1 / 2 / many, last token text / timestamp / EOT, previous token text / timestamp and
    last_ts -1 / ts_begin / mid-range / the last timestamp (floor + 1 = V removes every timestamp)."""
    text = lambda k: 1000 + 37 * k
    out = [[]]
    for n in (1, 2, 7, 40):
        for last_kind in ("text", "ts", "eot"):
            for prev_kind in (("text", "ts") if n >= 2 else (None,)):
                for lts in (None, ts_begin, ts_begin + 700, V - 1):
                    h = [text(k) for k in range(n)]
                    if last_kind == "ts":
                        if lts is None:
                            continue
                        h[-1] = lts
                    elif last_kind == "eot":
                        h[-1] = eot
                    if prev_kind == "ts":
                        if last_kind == "ts":
                            h[-2] = max(lts - 1, ts_begin)
                        elif lts is None:
                            continue
                        else:
                            h[-2] = lts
                    elif lts is not None and last_kind != "ts":
                        if n < 3:
                            continue
                        h[0] = lts
                    if n >= 7 and lts is not None and h[1] < ts_begin:
                        h[1] = ts_begin + 3                     # an earlier timestamp that does not set the floor
                    out.append(h)
    return out


@pytest.mark.parametrize("apply", [0, 1])
@pytest.mark.parametrize("max_init", [-1, 0, 50])
def test_every_compressed_state_gives_the_history_masks(apply, max_init):
    _gpu()
    tk, V = layout_tokenizer(True, 100)
    ids = _ids(tk)
    sup, first = _masks(tk, V)
    hs = _state_histories(ids["eot"], ids["ts_begin"], V)
    rng = np.random.default_rng(11 + apply * 7 + max_init)
    s = Sampler(ids, V, len(hs), 4, suppress=sup, first=first, apply=apply, max_init=max_init, histories=hs)
    s.step(np.stack([random_row(rng, V, ids["ts_begin"]) for _ in hs]))
    # the suppress mask alone, and the first-step mask alone (it applies at n_sampled == 0 only)
    for kw in (dict(suppress=sup), dict(first=first)):
        s = Sampler(ids, V, len(hs), 4, apply=apply, max_init=max_init, histories=hs, **kw)
        s.step(np.stack([random_row(rng, V, ids["ts_begin"]) for _ in hs]))
    print(f"apply_ts_rules={apply} max_initial_ts={max_init}: {len(hs)} states x 3 mask sets equal the history's masks")


def _scripts(ids, V, steps):
    """forced scripts [steps, 7]; ts(k) = ts_begin + k"""
    tb, eot = ids["ts_begin"], ids["eot"]
    ts = lambda k: tb + k
    x = lambda k: 500 + 97 * k
    rows = [
        [ts(10), x(1), x(2), ts(40), ts(40), x(3), ts(60), ts(70), x(4), ts(20), x(5), ts(90), ts(95), eot, x(6), x(7)],
        [ts(0), ts(5), x(1), ts(5), x(2), x(3), ts(30), x(4), x(5), ts(31), ts(31), x(6), x(7), x(8), eot, x(9)],
        [x(k) for k in range(12)] + [eot, x(1), x(2), x(3)],
        [x(1), x(2), ts(100), x(3), x(4), ts(200), x(5), ts(150), x(6), ts(150), ts(300), x(7), x(8), ts(400), ts(400), eot],
        [ts(1500), x(1), x(2), x(3), ts(1500), ts(1500), x(4), x(5), x(6), x(7), x(8), x(9), x(10), x(11), x(12), eot],
        [ts(0), ts(0), x(1), ts(2), ts(1), ts(3), x(2), ts(700), x(3), x(4), ts(699), x(5), ts(800), ts(900), x(6), eot],
        [x(k) for k in range(15)] + [eot],
    ]
    return np.array([r[:steps] for r in rows], dtype=np.int32).T.copy()


@pytest.mark.parametrize("T", [0.0, 0.7])
@pytest.mark.parametrize("tsmode", ["none", "shared", "rows1501", "rows1504"])
def test_forced_histories_step_by_step(T, tsmode):
    """16 forced steps + 2 past the step tables (argmax appended, nothing written), fresh logits at every step, compared
    against the restatement over the whole history after each step; row 2 is capped at 9 samples."""
    _gpu()
    tk, V = layout_tokenizer(True, 100)
    ids = _ids(tk)
    sup, first = _masks(tk, V)
    B, rows = 7, 16
    rng = np.random.default_rng(int(T * 10) * 10 + ["none", "shared", "rows1501", "rows1504"].index(tsmode))
    tsm, stride = None, 0
    if tsmode == "shared":
        tsm = rng.random(1501) < 0.2
    elif tsmode != "none":
        stride = 1501 if tsmode == "rows1501" else 1504
        tsm = rng.random((B, stride)) < 0.2
        tsm[:, 1501:] = True                                        # pitch padding: never read
    cap = np.full(B, 100, dtype=np.int32)
    cap[2] = 9
    s = Sampler(ids, V, B, rows, suppress=sup, first=first, ts_mask=tsm, ts_stride=stride, max_init=50, T=T,
                uniform=rng.random((rows, B)).astype(np.float32), cap=cap, forced=_scripts(ids, V, rows))
    for _ in range(rows + 2):
        s.step(np.stack([random_row(rng, V, ids["ts_begin"]) for _ in range(B)]))


@pytest.mark.parametrize("T", [0.0, 0.7, 1.0])
def test_free_running_draws_with_rules_on(T):
    """No forced tokens: the appended token is the kernel's own pick (argmax or inverse-CDF draw of the uniforms), under
    the timestamp rules; row 4 is capped at 5 samples, and 12 steps run against 10 table rows."""
    _gpu()
    tk, V = layout_tokenizer(True, 99)
    ids = _ids(tk)
    sup, first = _masks(tk, V)
    B, rows = 7, 10
    rng = np.random.default_rng(int(T * 10) + 3)
    u = rng.random((rows, B)).astype(np.float32)
    u[0, 0], u[1, 0] = 0.0, 1.0 - 2.0 ** -24
    cap = np.full(B, 50, dtype=np.int32)
    cap[4] = 5
    s = Sampler(ids, V, B, rows, suppress=sup, first=first, max_init=50, T=T, uniform=u, cap=cap)
    for _ in range(rows + 2):
        s.step(np.stack([random_row(rng, V, ids["ts_begin"]) for _ in range(B)]))


def test_timestamp_rule_margins_and_degenerate_rows():
    _gpu()
    tk, V = layout_tokenizer(True, 100)
    ids = _ids(tk)
    tb = ids["ts_begin"]
    rng = np.random.default_rng(21)
    xs, kinds = [], []
    for m in [1e-3, -1e-3] * 6 + [1e-8, -1e-8, 0.0] * 4:
        xs.append(random_row(rng, V, tb, tie_scale=m))
        kinds.append(m)
    for k in ("text", "ts", "all"):
        x = random_row(rng, V, tb)
        x[{"text": slice(0, tb), "ts": slice(tb, V), "all": slice(0, V)}[k]] = -np.inf
        xs.append(x)
        kinds.append(k)
    hs = [[600]] * len(xs)                                            # after one text token: no rule masks anything
    s = Sampler(ids, V, len(xs), 4, histories=hs)
    s.step(np.stack(xs))
    n_far = 0
    for x, k in zip(xs, kinds):
        if k in (1e-3, -1e-3):
            ref = restate(x, [600], **ids)
            assert ref["margin"] is not None and abs(ref["margin"]) > ref["band"], (k, ref["margin"], ref["band"])
            assert ref["kill_text"] == (k > 0)
            n_far += 1
    # the whole row -inf: nan_to_num makes it uniform, so the argmax is index 0 and its log-prob -log V
    assert int(s.nxt[-1]) == 0
    assert abs(float(s.states[-1:, 5].cpu().view(torch.float32)) + np.log(V)) < 1e-5
    print(f"{n_far} rows at +-1e-3 decided as in float64; near ties all-or-none; degenerate rows exact")


def test_special_values():
    _gpu()
    tk, V = layout_tokenizer(True, 100)
    ids = _ids(tk)
    tb, no_ts = ids["ts_begin"], ids["no_timestamps"]
    sup, first = _masks(tk, V)
    sup_idx = int(np.nonzero(sup)[0][3])
    rng = np.random.default_rng(31)

    def ts_heavy():                                    # timestamps clearly outweigh the text: the rule fires
        return random_row(rng, V, tb, tie_scale=3.0)

    free = np.nonzero(~sup[: ids["eot"]])[0]
    rows = []
    x = ts_heavy(); x[777] = np.nan; rows.append(x)                 # NaN among the text: no text may be suppressed
    x = ts_heavy(); x[tb + 9] = np.nan; rows.append(x)              # NaN among the timestamps
    x = ts_heavy(); x[no_ts] = np.nan; x[sup_idx] = np.nan; rows.append(x)   # NaN where a mask writes -inf
    x = ts_heavy(); x[1234] = np.inf; rows.append(x)                # +inf among the text
    x = random_row(rng, V, tb); x[tb + 44] = np.inf; rows.append(x)  # +inf among the timestamps
    x = random_row(rng, V, tb, tie_scale=-5.0)                      # an exact tie between two text tokens
    x[free[300]] = x[free[900]] = x[:tb].max() + 1.0
    rows.append(x)
    s = Sampler(ids, V, len(rows), 4, suppress=sup, first=first, histories=[[600]] * len(rows))
    out = s.step(np.stack(rows))
    assert (out[0, :tb] > -1e38).sum() > tb // 2, "NaN among the text logits: the text was suppressed"
    assert (out[2, :tb] < -1e38).all(), "NaN at masked indices: the timestamp rule must still suppress the text"
    assert int(s.nxt[5]) == free[300]
    # rules off: a tie between index 0 and index V - 1 goes to index 0
    x = random_row(rng, V, tb)
    x[0] = x[V - 1] = x.max() + 2.0
    s = Sampler(ids, V, 1, 4, apply=0, histories=[[600]])
    s.step(x[None])
    assert int(s.nxt[0]) == 0


SHAPES = [(lay, B) for lay in LAYOUTS + ["small"] for B in (1, 7, 300)]


@pytest.mark.parametrize("shape", SHAPES, ids=[f"V{51864 + LAYOUTS.index(l) if l != 'small' else 700}-B{B}" for l, B in SHAPES])
def test_shapes_vocabularies_and_padding(shape):
    """Random histories, per-row silent-timestamp masks, 3 steps at temperature 0.7; padding columns V..ld-1 (ld - V = 13)
    hold NaN sentinels.  The small V (700) leaves threads without indices in the temperature scan."""
    _gpu()
    layout, B = shape
    if layout == "small":
        V, ids = 700, dict(eot=300, ts_begin=304, no_timestamps=303)
        sup = np.zeros(V, dtype=bool); sup[[5, 301, 302]] = True
        first = np.zeros(V, dtype=bool); first[[32, 300]] = True
    else:
        tk, V = layout_tokenizer(*layout)
        ids = _ids(tk)
        sup, first = _masks(tk, V)
    rng = np.random.default_rng(V + B)
    hs = [random_history(rng, ids["eot"], ids["ts_begin"], V) for _ in range(B)]
    rows = max(len(h) for h in hs) + 3                        # every step of every row inside the tables
    s = Sampler(ids, V, B, rows, pad=13, suppress=sup, first=first, ts_mask=rng.random((B, 1501)) < 0.1, ts_stride=1501,
                max_init=50, T=0.7, uniform=rng.random((rows, B)).astype(np.float32), histories=hs)
    for _ in range(3):
        s.step(np.stack([random_row(rng, V, ids["ts_begin"]) for _ in range(B)]))


def test_report_worst_sum_logprob_error():
    _gpu()
    if WORST["ratio"] == 0.0:
        pytest.skip("run with the other tests of this file")
    print(f"worst sum_logprob |err| vs float64 {WORST['err']:.2e}, worst err / bound {WORST['ratio']:.3f} "
          f"(bound {SUM_LP_REL:g} * (|gmax| + |lse| + 1) per step)")
    assert WORST["ratio"] <= 1.0
