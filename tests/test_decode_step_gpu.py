"""The caption decoder's per-step kernels against HF's logits processors and fp64, one kernel at a time.

Every greedy decode step of the caption path runs ~70 launches.  Besides the end-to-end parity tests (a random stand-in
model, 6 crops, 20 tokens), this module pins each of them at the shapes the plans issue and at the edges where such
kernels go wrong:

* ``b2p_greedy_pick`` against ``transformers``' NoRepeatNGram / ForcedBOS / ForcedEOS processors + ``torch.argmax`` +
  the pad / EOS bookkeeping of HF's greedy loop, on crafted logits (ties, banned maxima, every n-gram size, ban lists
  longer than 64, forced steps with NaN logits, finished rows, odd vocabularies and pitches, unaligned rows, 1..416
  rows), through both scan paths (with and without a dump), and over whole generations of 20 and 250 steps;
* ``b2p_mha_cached`` over a whole decode (every step, every remainder of the four-key unroll, cache appends bit for bit);
* ``b2p_mha`` as the decoder's cross-attention and the 768-mode encoder's self-attention, against fp64;
* ``b2p_decoder_embed`` / ``b2p_encoder_embed`` / ``b2p_projector_prep`` bit for bit against float32 restatements;
* ``b2p_layernorm`` on its own against fp64 (large-mean and small-variance rows included);
* the decode step's GEMM calls (qkv, cross q, out-projections + residual, fc1 + GELU, fc2 + residual, LM head);
* on the CPU: every class of these calls the Florence plans issue has a case here, and the long-n-gram case really
  needs more than 64 bans.

Every launch stays inside its buffers: the extents are checked on the host before each call, and every buffer carries
finite guard values (rows / columns past what the kernel may write) that must be unchanged afterwards."""
from __future__ import annotations

import functools
import math
from dataclasses import dataclass

import pytest
import torch
import torch.nn.functional as F

from omniparser_b200 import ops
from test_parity_planes_gpu import _bits, _covers, _rejected, check_canonical, pair
from test_plan_dryrun_cpu import rec  # noqa: F401  (fixture: the C library replaced by an argument-checking recorder)

DEV = "cuda:0"
D, HEADS = 768, 12
EOS, PAD, BOS, START = 2, 1, 0, 2          # the Florence-2 generation config (standin/florence.py GEN)
SENTINEL = -1234.0                          # finite guard value, exactly representable in fp16 and fp32
SEQ_GUARD = -777                            # guard token id
LOGIT_GUARD = 1e30                          # finite, above every real logit: a read past V would win the argmax
TOL_X3 = 2e-5                               # fp16x3 pairs / split outputs, relative to max(1, |ref|max)
TOL_F16 = 1.5e-3                            # plain fp16 outputs
TOL_LN32 = 1e-5                             # fp32 LayerNorm
TOL_GEMM16 = 2e-3                           # fp16 GEMMs against fp32 on the rounded operands


def _tol(ref, rel):
    return rel * max(1.0, ref.abs().max().item())


def _same_bits(got, ref, what):
    got, ref = got.cpu(), ref.cpu()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    neq = _bits(got) != _bits(ref)
    assert not bool(neq.any()), f"{what}: {int(neq.sum())} elements differ"


def _act_value(o, C, split):
    """fp16 activation rows -> float64 values ([hi | lo] pairs summed)"""
    o = o.cpu().double()
    return o[:, :C] + o[:, C:2 * C] if split else o[:, :C]


# ================================================================================================ greedy_pick
# layout -> (V, logits row pitch, offset of the first row in floats)
LAYOUTS = {
    "v51290_ld51296": (51290, 51296, 0),       # the stand-in vocabulary in the plan's padded pitch: float2 vector path
    "v51289_ld51296": (51289, 51296, 0),       # a remote-code checkpoint: vector path, last id through the thread-0 tail
    "v51289_ld51289": (51289, 51289, 0),       # odd pitch: scalar path
    "v51290_ld51296_off1": (51290, 51296, 1),  # rows 4-byte but not 8-byte aligned: scalar path
    "v37_ld40": (37, 40, 0),                   # fewer ids than threads
}


@dataclass(frozen=True)
class PickParams:
    ngram: int = 3
    bos: int = BOS
    feos: int = EOS
    max_len: int = 21


def _noise(B, V, g):
    """base logits in [-1, 0): every crafted maximum below is >= 1"""
    return torch.rand(B, V, generator=g) - 1


def _rows(prefixes, V, g, tops, finished=None):
    """prefixes: per row the ids so far (all the same length); tops: per row {id: logit}"""
    n = len(prefixes[0])
    assert all(len(p) == n for p in prefixes)
    lg = _noise(len(prefixes), V, g)
    for b, top in enumerate(tops):
        for i, v in top.items():
            assert 0 <= i < V, (i, V)
            lg[b, i] = v
    fin = torch.tensor(finished if finished is not None else [0] * len(prefixes), dtype=torch.int32)
    return torch.tensor(prefixes, dtype=torch.long), fin, lg


def _long_prefix():
    """[2, 0] + 70 x (10, 11, 100 + i) + (10, 11): the (10, 11) prefix recurs 71 times, each time followed by a new id,
    so the next pick at length 214 must avoid 70 banned ids (100 .. 169)"""
    s = [START, BOS]
    for i in range(70):
        s += [10, 11, 100 + i]
    return s + [10, 11]


def _sc_tie_in_thread(V, g):
    # 10, 2058, 4106 are read by the same thread on both scan paths (float2 index 5 + 1024k; id 10 + 1024k)
    return _rows([[START, BOS, 5, 6]] * 2, V, g, [{10: 3.0, 2058: 3.0}, {2058: 3.0, 4106: 3.0}]), PickParams()


def _sc_tie_across_warps(V, g):
    # 1200 (vector thread 600, warp 18) ties 2058 (thread 5, warp 0): the lower index sits in the higher warp
    return _rows([[START, BOS, 5, 6]] * 3, V, g, [{10: 3.0, 200: 3.0}, {1200: 3.0, 2058: 3.0}, {40: 3.0, V - 1: 3.0}]), PickParams()


def _sc_tie_small(V, g):
    return _rows([[START, BOS, 5, 6]] * 2, V, g, [{3: 3.0, 33: 3.0}, {18: 3.0, 17: 3.0}]), PickParams()


def _sc_tie_float2_halves(V, g):
    return _rows([[START, BOS, 5, 6]] * 3, V, g, [{2000: 3.0, 2001: 3.0}, {2001: 3.0, 4049: 3.0}, {3: 3.0, 1002: 3.0}]), PickParams()


def _sc_tie_first_banned(V, g):
    # (7, 8) was followed by 300: 300 is banned, so the tie goes to the later id
    p = [START, BOS, 7, 8, 300, 9, 7, 8]
    return _rows([p, p], V, g, [{300: 3.0, 5000: 3.0}, {300: 3.0, 301: 3.0}]), PickParams()


def _sc_banned_max(V, g):
    # the maximum is banned; the runner-up sits in another warp.  Row 2: the last id is banned; row 3: the last id wins
    return _rows([[START, BOS, 7, 8, 64, 9, 7, 8], [START, BOS, 7, 8, 64, 9, 7, 8], [START, BOS, 7, 8, V - 1, 9, 7, 8],
                  [START, BOS, 7, 8, 64, 9, 7, 8]], V, g,
                 [{64: 5.0, 1400: 4.0}, {64: 5.0, 40000: 4.0, 3: 3.0}, {V - 1: 5.0, 33: 4.0}, {64: 5.0, V - 1: 4.0}]), PickParams()


def _sc_no_bans_yet(V, g):
    # cur_len + 1 < ngram: nothing is banned, not even a repeated id
    return _rows([[START, 7], [START, START]], V, g, [{7: 3.0, 9: 2.0}, {START: 3.0}]), PickParams(ngram=4, bos=-1)


_FILL = [40, 41, 42, 43, 44, 45]      # distinct filler ids: they complete no n-gram


def _sc_ngram(k):
    def build(V, g):
        # row 0: the only ban comes from the n-gram that starts at s = cur_len - ngram (ends at the last position);
        # row 1: the (k-1)-gram prefix occurred twice before, followed by 12 and by 13
        if k == 1:
            r0, r1 = [START, BOS, 9, 7], [START, BOS, 12, 13]
            tops = [{7: 6.0, 9: 5.5, 21: 5.0}, {12: 6.0, 13: 5.5, START: 5.1, BOS: 5.05, 21: 5.0}]
        else:
            pre = [9, 10, 11][3 - (k - 1):]
            r1 = [START, BOS] + pre + [12] + pre + [13] + pre
            r0 = [START, BOS] + _FILL[:len(r1) - 3 - k] + [6] + [5] * k
            tops = [{5: 6.0, 21: 5.0}, {12: 6.0, 13: 5.5, 21: 5.0}]
        return _rows([r0, r1], V, g, tops), PickParams(ngram=k)
    return build


def _sc_long_ngram(V, g):
    p = _long_prefix()
    # row 0: the top id is the 70th ban, the second the 66th; row 1: the top id is the first ban
    return _rows([p, p], V, g, [{169: 6.0, 165: 5.5, 40000: 5.0}, {100: 6.0, 40001: 5.0}]), PickParams(max_len=250)


def _sc_long_ngram1(V, g):
    # ngram = 1 bans every id seen so far: 202 of them
    p = [START, BOS] + [300 + i for i in range(200)]
    return _rows([p], V, g, [{499: 6.0, 450: 5.5, 250: 5.0}]), PickParams(ngram=1, max_len=250)


def _sc_forced_bos(V, g):
    return _rows([[START]] * 3, V, g, [{V - 1: 5.0}, {7: 5.0}, {EOS: 5.0}], finished=[0, 1, 0]), PickParams()


def _sc_forced_eos(V, g):
    pre = [START, BOS] + [30 + i for i in range(18)]           # length 20 = max_len - 1
    return _rows([pre] * 3, V, g, [{V - 1: 5.0}, {7: 5.0}, {EOS: -5.0}], finished=[0, 1, 0]), PickParams()


def _sc_forced_bos_nan(V, g):
    (ids, fin, lg), p = _sc_forced_bos(V, g)
    return (ids, fin, torch.full_like(lg, float("nan"))), p


def _sc_forced_eos_nan(V, g):
    (ids, fin, lg), p = _sc_forced_eos(V, g)
    return (ids, fin, torch.full_like(lg, float("nan"))), p


def _sc_finished_rows(V, g):
    p = [START, BOS, 5, 6]
    return _rows([p] * 4, V, g, [{9: 3.0}, {EOS: 3.0}, {11: 3.0}, {12: 3.0}], finished=[0, 1, 0, 1]), PickParams()


def _sc_picks_eos(V, g):
    # rows 0 and 3 pick EOS (row 3 in a tie with a later id) and finish; row 1 would pick EOS but is already finished
    p = [START, BOS, 5, 6]
    return _rows([p] * 4, V, g, [{EOS: 3.0}, {EOS: 3.0}, {9: 3.0}, {EOS: 3.0, 20: 3.0}], finished=[0, 1, 0, 0]), PickParams()


def _sc_rows(B):
    def build(V, g):
        # ids from a 6-token alphabet so that bans fire; the top of each row is often a banned id or EOS
        ids = torch.randint(3, 9, (B, 12), generator=g)
        ids[:, 0], ids[:, 1] = START, BOS
        lg = _noise(B, V, g)
        lg[:, 2:12] += torch.rand(B, 10, generator=g) * 4 + 1
        lg[:, EOS] += (torch.rand(B, generator=g) < 0.2).float() * 8
        fin = (torch.rand(B, generator=g) < 0.2).int()
        return (ids, fin, lg), PickParams()
    return build


PICK_SCENARIOS = {
    "tie_in_thread": (_sc_tie_in_thread, 4107),
    "tie_across_warps": (_sc_tie_across_warps, 2059),
    "tie_float2_halves": (_sc_tie_float2_halves, 4050),
    "tie_small": (_sc_tie_small, 34),
    "tie_first_banned": (_sc_tie_first_banned, 5001),
    "banned_max": (_sc_banned_max, 40001),
    "no_bans_yet": (_sc_no_bans_yet, 10),
    "ngram1": (_sc_ngram(1), 46),
    "ngram2": (_sc_ngram(2), 46),
    "ngram3": (_sc_ngram(3), 46),
    "ngram4": (_sc_ngram(4), 46),
    "long_ngram": (_sc_long_ngram, 40002),
    "long_ngram1": (_sc_long_ngram1, 500),
    "forced_bos": (_sc_forced_bos, 8),
    "forced_eos": (_sc_forced_eos, 48),
    "forced_bos_nan": (_sc_forced_bos_nan, 8),
    "forced_eos_nan": (_sc_forced_eos_nan, 48),
    "finished_rows": (_sc_finished_rows, 13),
    "picks_eos": (_sc_picks_eos, 21),
    "rows1": (_sc_rows(1), 13),
    "rows7": (_sc_rows(7), 13),
    "rows416": (_sc_rows(416), 13),
}
PICK_CASES = [(s, l) for s, (_, vmin) in PICK_SCENARIOS.items() for l, (V, _, _) in LAYOUTS.items() if V >= vmin]
LONG_NGRAM = {"long_ngram", "long_ngram1"}      # ban lists longer than 64


@functools.lru_cache(maxsize=None)
def pick_case(scen, V):
    g = torch.Generator().manual_seed(sum(map(ord, scen)) + V)
    (ids, fin, lg), p = PICK_SCENARIOS[scen][0](V, g)
    return ids, fin, lg.float().contiguous(), p


def hf_pick(ids, scores, finished, p: PickParams):
    """One step of HF's greedy loop: the processors in the order GenerationMixin._get_logits_processor builds them,
    argmax (first maximum), pad for finished rows, EOS bookkeeping (hf:generation/utils.py:2727-2805).
    -> (next ids [B], finished after the step [B], processed scores [B, V])"""
    from transformers import ForcedBOSTokenLogitsProcessor, ForcedEOSTokenLogitsProcessor, NoRepeatNGramLogitsProcessor
    s = scores.clone()
    if p.ngram > 0:
        s = NoRepeatNGramLogitsProcessor(p.ngram)(ids, s)
    if p.bos >= 0:
        s = ForcedBOSTokenLogitsProcessor(p.bos)(ids, s)
    if p.feos >= 0:
        s = ForcedEOSTokenLogitsProcessor(p.max_len, p.feos)(ids, s)
    nxt = torch.argmax(s, -1)
    unfinished = 1 - finished.long()
    nxt = nxt * unfinished + PAD * (1 - unfinished)
    return nxt, finished.long() | (nxt == EOS).long(), s


def capped_pick(ids, scores, p: PickParams, cap=64):
    """The pick with the ban list truncated to its first `cap` entries in start-position order (what a fixed-size list
    keeps), for the non-forced steps of row 0"""
    row = ids[0].tolist()
    n, pre = len(row), p.ngram - 1
    bans = [row[s + pre] for s in range(n - p.ngram + 1) if row[s:s + pre] == row[n - pre:]]
    s = scores[0].clone()
    s[bans[:cap]] = -math.inf
    return int(torch.argmax(s)), len(bans)


def issue_pick(scen, layout, dump, dev, counter=True):
    """device buffers of one case (every guard filled), extents checked; launches b2p_greedy_pick -> buffers"""
    V, ld, off = LAYOUTS[layout]
    ids, fin, lg, p = pick_case(scen, V)
    B, cur_len = ids.shape
    seq_ld = p.max_len + 4                          # guard columns past the plan's max_len + 1
    assert 1 <= cur_len <= p.max_len - 1 and cur_len < seq_ld
    seq = torch.full((B, seq_ld), SEQ_GUARD, dtype=torch.int32)
    seq[:, :cur_len] = ids.int()
    flat = torch.full((off + (B + 1) * ld,), LOGIT_GUARD)    # + one guard row, and the pitch padding
    rows = flat[off:off + B * ld].view(B, ld)
    rows[:, :V] = lg
    finished = torch.cat([fin, torch.tensor([7], dtype=torch.int32)])
    n0 = int((fin == 0).sum())
    cnt = torch.tensor([n0, 99], dtype=torch.int32)
    dmp = torch.full(((B + 1) * V,), SENTINEL) if dump else None
    step = torch.tensor([cur_len - 1], dtype=torch.int32)
    t = {k: (v.to(dev) if v is not None else None) for k, v in dict(seq=seq, flat=flat, finished=finished, cnt=cnt, dump=dmp, step=step).items()}
    lrows = t["flat"][off:off + B * ld].view(B, ld)
    _covers(t["flat"], lrows.data_ptr(), (B - 1) * ld + V)
    _covers(t["seq"], t["seq"].data_ptr(), B * seq_ld)
    if dump:
        _covers(t["dump"], t["dump"].data_ptr(), B * V)
    ops.greedy_pick(lrows, ld, V, B, t["seq"], seq_ld, t["finished"], t["step"], p.ngram, p.bos, p.feos, EOS, PAD, p.max_len,
                    t["dump"], t["cnt"] if counter else None)
    return t, dict(seq=seq, flat=flat, finished=finished, cnt=cnt, dump=dmp, n0=n0, B=B, V=V, cur_len=cur_len)


def check_pick(scen, layout, dump, counter=True):
    t, h = issue_pick(scen, layout, dump, DEV, counter)
    torch.cuda.synchronize()
    ids, fin, lg, p = pick_case(scen, h["V"])
    B, V, cur_len = h["B"], h["V"], h["cur_len"]
    nxt, fin_ref, proc = hf_pick(ids, lg, fin, p)
    path = "scalar path (dump)" if dump else "production path (no dump)"
    seq = t["seq"].cpu()
    got = seq[:, cur_len].long()
    bad = (got != nxt).nonzero().flatten().tolist()
    assert not bad, f"{path}: rows {bad[:8]} picked {got[bad[:8]].tolist()}, HF picks {nxt[bad[:8]].tolist()}"
    exp_seq = h["seq"].clone()
    exp_seq[:, cur_len] = nxt.int()
    _same_bits(seq, exp_seq, f"{path}: seq outside column {cur_len}")
    _same_bits(t["finished"], torch.cat([fin_ref.int(), torch.tensor([7], dtype=torch.int32)]), f"{path}: finished")
    n_new = int(((fin_ref == 1) & (fin == 0)).sum())
    _same_bits(t["cnt"], torch.tensor([h["n0"] - n_new if counter else h["n0"], 99], dtype=torch.int32), f"{path}: n_unfinished")
    _same_bits(t["flat"], h["flat"], f"{path}: logits buffer")
    if dump:
        _same_bits(t["dump"][:B * V].view(B, V), proc, f"{path}: dump vs HF processed scores")
        _same_bits(t["dump"][B * V:], h["dump"][B * V:], f"{path}: dump guard row")


@pytest.mark.gpu
@pytest.mark.parametrize("scen,layout", PICK_CASES, ids=[f"{s}-{l}" for s, l in PICK_CASES])
def test_greedy_pick_vs_hf_processors(scen, layout):
    for dump in (False, True):
        check_pick(scen, layout, dump)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["v51290_ld51296", "v51289_ld51289"])
def test_greedy_pick_without_counter(layout):
    """n_unfinished = None: rows still finish, nothing else is written"""
    for dump in (False, True):
        check_pick("picks_eos", layout, dump, counter=False)


# ---------------------------------------------------------------------------------------- greedy loop
LOOP_B = 6


def loop_finish_steps(T):
    """per row: the step at which EOS gets the top logit (rows 4, 5 run until the forced EOS of the last step)"""
    return [3, T // 3, T // 2, T - 3, T + 10, T + 10]


def loop_logits(hf_seq, t, T, V, seed):
    """Row b favours the cycle a_b, c_b, X_b(i): after c_b the X ids score 4 - 0.001 i, so the pick is the first X that
    is not banned yet.  The (a_b, c_b) prefix recurs every three steps followed by a new X, so the ban list grows by one
    each cycle (83 entries by step 250).  EOS tops the row at its finish step."""
    g = torch.Generator().manual_seed(seed * 100003 + t)
    lg = _noise(LOOP_B, V, g)
    fin_at = loop_finish_steps(T)
    for b in range(LOOP_B):
        a, c = 20 + 2 * b, 21 + 2 * b
        last = int(hf_seq[b, -1])
        if t == fin_at[b]:
            lg[b, EOS] = 10.0
        elif last == a:
            lg[b, c] = 5.0
        elif last == c:
            x0 = 1000 + 400 * b
            lg[b, x0:x0 + 400] = 4.0 - 0.001 * torch.arange(400, dtype=torch.float32)
        else:
            lg[b, a] = 5.0
    return lg


def loop_buffers(T, dump, dev):
    V, ld = 51290, 51296
    max_len = T + 1
    seq_ld = max_len + 1                                  # the plan's layout
    t = dict(seq=torch.full((LOOP_B, seq_ld), 0, dtype=torch.int32), logits=torch.full((LOOP_B + 1, ld), LOGIT_GUARD),
             finished=torch.zeros(LOOP_B, dtype=torch.int32), cnt=torch.tensor([LOOP_B], dtype=torch.int32),
             step=torch.zeros(1, dtype=torch.int32), dump=torch.full((LOOP_B, V), SENTINEL) if dump else None)
    t["seq"][:, 0] = START
    return {k: (v.to(dev) if v is not None else None) for k, v in t.items()}, V, ld, max_len, seq_ld


def loop_pick(t, V, ld, max_len, seq_ld):
    ops.greedy_pick(t["logits"], ld, V, LOOP_B, t["seq"], seq_ld, t["finished"], t["step"], 3, BOS, EOS, EOS, PAD, max_len,
                    t["dump"], t["cnt"])


@pytest.mark.gpu
@pytest.mark.parametrize("T", [20, 250])
@pytest.mark.parametrize("dump", [False, True])
def test_greedy_loop_vs_hf(T, dump):
    """greedy_pick + step_advance for T steps against HF's loop: bans fire every cycle, rows finish at different steps"""
    t, V, ld, max_len, seq_ld = loop_buffers(T, dump, DEV)
    p = PickParams(max_len=max_len)
    hf_seq = torch.full((LOOP_B, 1), START, dtype=torch.long)
    hf_fin = torch.zeros(LOOP_B, dtype=torch.long)
    most_bans = 0
    for step in range(T):
        lg = loop_logits(hf_seq, step, T, V, seed=T)
        t["logits"][:LOOP_B, :V].copy_(lg)
        assert step + 1 < seq_ld and step + 1 <= max_len - 1
        loop_pick(t, V, ld, max_len, seq_ld)
        ops.step_advance(t["step"])
        nxt, hf_fin_new, _ = hf_pick(hf_seq, lg, hf_fin, p)
        most_bans = max(most_bans, capped_pick(hf_seq[-1:], lg[-1:], p)[1])     # row 5 runs to the end
        hf_seq = torch.cat([hf_seq, nxt[:, None]], 1)
        torch.cuda.synchronize()
        got = t["seq"][:, step + 1].cpu().long()
        assert torch.equal(got, nxt), f"step {step}: picked {got.tolist()}, HF picks {nxt.tolist()}"
        hf_fin = hf_fin_new
        assert torch.equal(t["finished"].cpu().long(), hf_fin), f"step {step}: finished"
        assert int(t["cnt"].item()) == LOOP_B - int(hf_fin.sum()), f"step {step}: n_unfinished"
    assert int(t["step"].item()) == T
    assert torch.equal(t["seq"][:, :T + 1].cpu().long(), hf_seq)
    assert int(t["seq"][:, T + 1].abs().sum()) == 0                 # the spare column is never written
    assert bool((t["logits"][LOOP_B] == LOGIT_GUARD).all())
    fin_steps = loop_finish_steps(T)
    assert len({s for s in fin_steps if s < T - 1}) >= 3 and bool(hf_fin.all())
    assert most_bans > (64 if T > 200 else 0)


# ---------------------------------------------------------------------------------------- argument checks
@pytest.mark.gpu
def test_greedy_pick_rejects_arguments_it_cannot_honour():
    """Every buffer is large enough for the call as written; the C side must still refuse each call before launching."""
    from omniparser_b200 import _lib
    B, V, max_len = 2, 64, 21
    logits = torch.zeros(B, 2 * V, device=DEV)
    seq = torch.full((B * 9000,), SEQ_GUARD, dtype=torch.int32, device=DEV)
    fin = torch.zeros(B, dtype=torch.int32, device=DEV)
    step = torch.zeros(1, dtype=torch.int32, device=DEV)
    cnt = torch.tensor([B], dtype=torch.int32, device=DEV)
    good = dict(V=V, ld=V, B=B, seq_ld=max_len + 1, ngram=3, bos=BOS, feos=EOS, max_len=max_len)

    def call(**kw):
        a = {**good, **kw}
        ops.greedy_pick(logits, a["ld"], a["V"], a["B"], seq, a["seq_ld"], fin, step, a["ngram"], a["bos"], a["feos"], EOS, PAD,
                        a["max_len"], None, cnt)
    _rejected(lambda: call(V=0), "V <= ld")
    _rejected(lambda: call(ld=V - 1), "V <= ld")
    _rejected(lambda: call(ngram=-1), "ngram")
    _rejected(lambda: call(max_len=1, seq_ld=2), "max_len")
    _rejected(lambda: call(max_len=8193, seq_ld=8194), "max_len")
    _rejected(lambda: call(seq_ld=max_len - 1), "seq_ld")
    _rejected(lambda: call(bos=V), "forced token")
    _rejected(lambda: call(feos=V), "forced token")
    _rejected(lambda: call(B=-1), "B must be")
    n0 = _lib.launch_count()
    call(B=0)                                             # nothing to do: no launch, no error
    assert _lib.launch_count() == n0
    call(max_len=8192, seq_ld=8192)                       # the largest ban list (32 KiB of shared memory); step 0: forced BOS
    torch.cuda.synchronize()
    assert _lib.launch_count() == n0 + 1
    assert seq[1].item() == BOS and seq[8192 + 1].item() == BOS


# ================================================================================================ mha_cached
def _attn_ref(q, k, v):
    """fp64 softmax attention, q [..., Lq, 64] (unscaled), k / v [..., Lk, 64]"""
    return torch.softmax((q.double() * 0.125) @ k.double().transpose(-1, -2), -1) @ v.double()


SPIKES = (5, 6, 13, 30, 47)      # steps whose key scores far above every earlier key: the online-softmax rescale


def issue_mha_cached(t, qkv, kc, vc, tmax, step, R, out, split):
    assert 0 <= t < tmax and qkv.shape == (R, 3 * D) and kc.shape[1] == tmax and kc.shape[0] > R
    _covers(qkv, qkv.data_ptr(), R * 3 * D)
    _covers(kc, kc.data_ptr(), R * tmax * D); _covers(vc, vc.data_ptr(), R * tmax * D)
    _covers(out, out.data_ptr(), R * out.shape[1])
    ops.mha_cached(qkv, 3 * D, qkv[:, D:], qkv[:, 2 * D:], 3 * D, kc, vc, tmax, step, R, HEADS, out, out.stride(0), split=split)


def mha_cached_buffers(R, tmax, split, dev):
    return (torch.zeros(R, 3 * D, device=dev), torch.full((R + 1, tmax, D), SENTINEL, device=dev),
            torch.full((R + 1, tmax, D), SENTINEL, device=dev), torch.zeros(1, dtype=torch.int32, device=dev),
            torch.full((R + 1, (2 if split else 1) * D), SENTINEL, dtype=torch.float16, device=dev))


MHA_CACHED_CASES = [(tmax, R, split) for tmax in (21, 64) for R in (2, 6, 32) for split in (False, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("tmax,R,split", MHA_CACHED_CASES)
def test_mha_cached_whole_decode(tmax, R, split):
    """decoder self-attention over a whole decode: step t appends k / v at cache row t and attends over rows 0..t"""
    g = torch.Generator().manual_seed(tmax * 100 + R * 2 + split)
    qkv, kc, vc, step, out = mha_cached_buffers(R, tmax, split, DEV)
    qbase = torch.randn(R, HEADS, 64, generator=g)
    ks, vs = [], []
    for t in range(tmax):
        q = qbase + 0.3 * torch.randn(R, HEADS, 64, generator=g)
        k = 0.5 * torch.randn(R, HEADS, 64, generator=g) + (3.0 if t in SPIKES else 0.0) * qbase
        v = torch.randn(R, HEADS, 64, generator=g)
        qkv.copy_(torch.cat([q.reshape(R, D), k.reshape(R, D), v.reshape(R, D)], 1))
        step.fill_(t)
        issue_mha_cached(t, qkv, kc, vc, tmax, step, R, out, split)
        torch.cuda.synchronize()
        ks.append(k.reshape(R, D)); vs.append(v.reshape(R, D))
        K, V_ = torch.stack(ks, 1), torch.stack(vs, 1)          # [R, t+1, D]
        kch, vch = kc.cpu(), vc.cpu()
        _same_bits(kch[:R, :t + 1], K, f"step {t}: k cache rows 0..t")
        _same_bits(vch[:R, :t + 1], V_, f"step {t}: v cache rows 0..t")
        assert bool((kch[:R, t + 1:] == SENTINEL).all() and (vch[:R, t + 1:] == SENTINEL).all()), f"step {t}: cache rows > t written"
        assert bool((kch[R] == SENTINEL).all() and (vch[R] == SENTINEL).all()), f"step {t}: guard batch row written"
        ref = _attn_ref(q.reshape(R, HEADS, 1, 64), K.view(R, t + 1, HEADS, 64).transpose(1, 2),
                        V_.view(R, t + 1, HEADS, 64).transpose(1, 2)).reshape(R, D)
        o = out.cpu()
        err, tol = (_act_value(o[:R], D, split) - ref).abs().max().item(), _tol(ref, TOL_X3 if split else TOL_F16)
        assert err < tol, f"step {t}: max abs err {err:.3g} > {tol:.3g}"
        if split:
            check_canonical(o[:R, :D], o[:R, D:])
        assert bool((o[R] == SENTINEL).all()), f"step {t}: guard output row written"


# ================================================================================================ mha (first version)
# name -> (Lq, Lk, v3 flag as the plan passes it); cross: q [R, 768], kv [R*Lk, 1536] with v at column 768;
# self: qkv [R*L, 2304]
MHA_CASES = {
    "cross_L13": (1, 13, False),
    "cross_L585": (1, 585, False),
    "self_L585_v3flag": (585, 585, True),      # 768-mode encoder: L > 16, the v3 flag falls through to mha_kernel
    "self_L13_v3": (13, 13, True),             # 64-mode encoder: the warp-per-head kernel
}
MHA_ROWS = [("cross_L13", 2), ("cross_L13", 6), ("cross_L13", 32), ("cross_L585", 2), ("cross_L585", 6),
            ("self_L585_v3flag", 2), ("self_L13_v3", 6)]


def issue_mha(name, R, split, dev):
    Lq, Lk, v3 = MHA_CASES[name]
    g = torch.Generator().manual_seed(sum(map(ord, name)) + R + split)
    out = torch.full((R * Lq + 1, (2 if split else 1) * D), SENTINEL, dtype=torch.float16)
    if Lq == 1:
        q = torch.randn(R, D, generator=g)
        kv = torch.randn(R * Lk, 2 * D, generator=g)
        q, kv, out = q.to(dev), kv.to(dev), out.to(dev)
        _covers(q, q.data_ptr(), R * D); _covers(kv, kv.data_ptr(), R * Lk * 2 * D)
        args = (q, D, kv, kv[:, D:], 2 * D)
        host = (q.cpu().view(R, 1, HEADS, 64), kv.cpu()[:, :D].reshape(R, Lk, HEADS, 64), kv.cpu()[:, D:].reshape(R, Lk, HEADS, 64))
    else:
        qkv = torch.randn(R * Lq, 3 * D, generator=g).to(dev)
        out = out.to(dev)
        _covers(qkv, qkv.data_ptr(), R * Lq * 3 * D)
        args = (qkv, 3 * D, qkv[:, D:], qkv[:, 2 * D:], 3 * D)
        h = qkv.cpu().view(R, Lq, 3, HEADS, 64)
        host = (h[:, :, 0], h[:, :, 1], h[:, :, 2])
    _covers(out, out.data_ptr(), R * Lq * out.shape[1])
    ops.mha(*args, R, Lq, Lk, HEADS, out, out.stride(0), split=split, v3=v3)
    return out, host


@pytest.mark.gpu
@pytest.mark.parametrize("name,R", MHA_ROWS)
@pytest.mark.parametrize("split", [False, True])
def test_mha_vs_fp64(name, R, split):
    Lq, Lk, _ = MHA_CASES[name]
    out, (q, k, v) = issue_mha(name, R, split, DEV)
    torch.cuda.synchronize()
    ref = _attn_ref(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)).transpose(1, 2).reshape(R * Lq, D)
    o = out.cpu()
    err, tol = (_act_value(o[:R * Lq], D, split) - ref).abs().max().item(), _tol(ref, TOL_X3 if split else TOL_F16)
    assert err < tol, f"max abs err {err:.3g} > {tol:.3g}"
    assert bool((o[R * Lq] == SENTINEL).all())


# ================================================================================================ embeddings
DEC_VOCAB, N_POS = 51290, 1026          # BART: 1024 learned positions + offset 2


@functools.lru_cache(maxsize=None)
def embed_tables(dev):
    g = torch.Generator().manual_seed(11)
    return torch.randn(DEC_VOCAB, D, generator=g).to(dev), torch.randn(N_POS, D, generator=g).to(dev)


DEC_EMBED_CASES = [(max_len, extra, which) for max_len in (21, 1025) for extra in (1, 9) for which in ("first", "middle", "last")]


def issue_decoder_embed(max_len, extra, which, dev):
    E, P = embed_tables(dev)
    B, seq_ld = 6, max_len + extra
    t = {"first": 0, "middle": max_len // 2, "last": max_len - 2}[which]
    assert t < seq_ld and t + 2 < N_POS
    g = torch.Generator().manual_seed(max_len + extra + t)
    seq = torch.randint(0, DEC_VOCAB, (B, seq_ld), generator=g, dtype=torch.int32)
    seq[0, t] = DEC_VOCAB - 1
    seq_d, step = seq.to(dev), torch.tensor([t], dtype=torch.int32, device=dev)
    out = torch.full((B + 1, D), SENTINEL, device=dev)
    ops.decoder_embed(E, seq_d, seq_ld, step, P, B, D, out)
    return out, seq, t


@pytest.mark.gpu
@pytest.mark.parametrize("max_len,extra,which", DEC_EMBED_CASES)
def test_decoder_embed_bit_exact(max_len, extra, which):
    out, seq, t = issue_decoder_embed(max_len, extra, which, DEV)
    torch.cuda.synchronize()
    E, P = embed_tables("cpu")
    ref = E[seq[:, t].long()] + P[t + 2]
    _same_bits(out[:-1], ref, f"decoder_embed step {t}")
    assert bool((out[-1] == SENTINEL).all())


def issue_encoder_embed(n_img, B, dev):
    from standin.florence import PROMPT_IDS
    E, P = embed_tables(dev)
    g = torch.Generator().manual_seed(n_img + B)
    img = torch.randn(B, n_img, D, generator=g).to(dev)
    prompt = torch.tensor(PROMPT_IDS, dtype=torch.int32, device=dev)
    L = n_img + len(PROMPT_IDS)
    assert L + 1 < N_POS
    out = torch.full((B * L + 1, D), SENTINEL, device=dev)
    ops.encoder_embed(img, n_img, E, prompt, len(PROMPT_IDS), P, B, D, out)
    return out, img, prompt


@pytest.mark.gpu
@pytest.mark.parametrize("n_img,B", [(5, 6), (577, 2)])
def test_encoder_embed_bit_exact(n_img, B):
    out, img, prompt = issue_encoder_embed(n_img, B, DEV)
    torch.cuda.synchronize()
    E, P = embed_tables("cpu")
    n_p = prompt.numel()
    rows = torch.cat([img.cpu(), E[prompt.cpu().long()].expand(B, n_p, D)], 1) + P[2:2 + n_img + n_p]
    _same_bits(out[:-1], rows.reshape(-1, D), "encoder_embed")
    assert bool((out[-1] == SENTINEL).all())


# ================================================================================================ projector_prep
def issue_projector_prep(HW, split, dev, B=3, C=1024):
    g = torch.Generator().manual_seed(HW * 2 + split)
    x = (torch.randn(B, HW, C, generator=g) * 2 + 0.5).to(dev)
    pos = torch.randn(HW, C, generator=g).to(dev)
    out = torch.full((B * (HW + 1) + 1, (2 if split else 1) * C), SENTINEL, dtype=torch.float16, device=dev)
    ops.projector_prep(x, pos, B, HW, C, out, split=split)
    return out, x, pos


@pytest.mark.gpu
@pytest.mark.parametrize("HW", [4, 576])
@pytest.mark.parametrize("split", [False, True])
def test_projector_prep_bit_exact(HW, split):
    B, C = 3, 1024
    out, x, pos = issue_projector_prep(HW, split, DEV)
    torch.cuda.synchronize()
    v = x.cpu() + pos.cpu()                                  # [B, HW, C] fp32, one rounding
    s = torch.zeros(B, C)
    for t in range(HW):                                      # the kernel's sequential fp32 sum
        s = s + v[:, t]
    mean = s / torch.full_like(s, HW)
    rows = torch.cat([mean[:, None], v], 1).reshape(-1, C)   # [B*(HW+1), C]: mean row, then the tokens
    o = out.cpu()
    if split:
        hi, lo = pair(rows)
        _same_bits(o[:-1, :C], hi, "hi plane"); _same_bits(o[:-1, C:], lo, "lo plane")
    else:
        _same_bits(o[:-1], rows.half(), "fp16 rows")
    ref = x.cpu().double().add(pos.cpu().double()).mean(1)
    got = _act_value(o[:-1], C, split).view(B, HW + 1, C)[:, 0]
    assert (got - ref).abs().max().item() < _tol(ref, TOL_X3 if split else TOL_F16)
    assert bool((o[-1] == SENTINEL).all())


# ================================================================================================ layernorm
LN_CS = [128, 256, 512, 768, 1024, 200]           # 200: not a multiple of 128 (lanes hold 2 or 1 float4)
LN_OUTS = ["out16", "out32", "both"]
LN_SCALES = {"unit": (0.0, 1.0), "mean100": (100.0, 1.0), "small_var": (0.0, 3e-3)}   # small_var: eps matters


def issue_layernorm(C, outs, split, scale, dev, T=37):
    g = torch.Generator().manual_seed(C + T + 7 * split + len(outs) + int(LN_SCALES[scale][1] * 1000))
    m, s = LN_SCALES[scale]
    x = (torch.randn(T, C, generator=g) * s + m).to(dev)
    gam, bet = torch.randn(C, generator=g).to(dev), torch.randn(C, generator=g).to(dev)
    o16 = torch.full((T + 1, (2 if split else 1) * C), SENTINEL, dtype=torch.float16, device=dev) if outs != "out32" else None
    o32 = torch.full((T + 1, C), SENTINEL, device=dev) if outs != "out16" else None
    ops.layernorm(x, gam, bet, T, C, o16, o32, split=split)
    return x, gam, bet, o16, o32


@pytest.mark.gpu
@pytest.mark.parametrize("C", LN_CS)
@pytest.mark.parametrize("outs", LN_OUTS)
@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("scale", list(LN_SCALES))
def test_layernorm_vs_fp64(C, outs, split, scale):
    """T = 37 rows: not a multiple of the 8 rows (warps) per CTA"""
    x, gam, bet, o16, o32 = issue_layernorm(C, outs, split, scale, DEV)
    torch.cuda.synchronize()
    ref = F.layer_norm(x.cpu().double(), (C,), gam.cpu().double(), bet.cpu().double(), 1e-5)
    if o32 is not None:
        y = o32.cpu()
        err, tol = (y[:-1].double() - ref).abs().max().item(), _tol(ref, TOL_LN32)
        assert err < tol, f"out32: max abs err {err:.3g} > {tol:.3g}"
        assert bool((y[-1] == SENTINEL).all())
    if o16 is not None:
        h = o16.cpu()
        err, tol = (_act_value(h[:-1], C, split) - ref).abs().max().item(), _tol(ref, TOL_X3 if split else TOL_F16)
        assert err < tol, f"out16: max abs err {err:.3g} > {tol:.3g}"
        assert bool((h[-1] == SENTINEL).all())
        if o32 is not None:              # out16 is the rounding of out32: the canonical pair, or plain fp16
            if split:
                hi, lo = pair(o32.cpu()[:-1])
                _same_bits(h[:-1, :C], hi, "out16 hi vs out32"); _same_bits(h[:-1, C:], lo, "out16 lo vs out32")
            else:
                _same_bits(h[:-1], o32.cpu()[:-1].half(), "out16 vs out32")


# ================================================================================================ decode-step GEMMs
# kind -> (N, K, bias, residual, act, output): exactly the calls FlorencePlan._build_dec_part issues
GEMM_KINDS = {
    "qkv": (3 * D, D, True, False, ops.ACT_NONE, "f32"),
    "cross_q": (D, D, True, False, ops.ACT_NONE, "f32"),
    "out_proj_res": (D, D, True, True, ops.ACT_NONE, "f32"),       # self out-proj and cross out-proj
    "fc1_gelu": (4 * D, D, True, False, ops.ACT_GELU, "f16"),       # fp16x3 mode: [hi | lo] output
    "fc2_res": (D, 4 * D, True, True, ops.ACT_NONE, "f32"),
    "lm_head": (51290, D, False, False, ops.ACT_NONE, "logits"),   # into the padded pitch 51296
}
GEMM_CASES = [(k, prec, M) for k in GEMM_KINDS for prec in ("fp16x3", "fp16") for M in (2, 6, 32)]


@functools.lru_cache(maxsize=None)
def gemm_weights(kind, prec):
    N, K, has_bias, *_ = GEMM_KINDS[kind]
    g = torch.Generator().manual_seed(sum(map(ord, kind)))
    w32 = torch.randn(N, K, generator=g) / math.sqrt(K)
    bias = torch.randn(N, generator=g) * 0.5 if has_bias else None
    hi, lo = pair(w32)
    w = torch.cat([hi, lo], 1).contiguous() if prec == "fp16x3" else hi.contiguous()
    wref = hi.double() + lo.double() if prec == "fp16x3" else hi.double()
    return w, wref, bias


def issue_gemm(kind, prec, M, dev):
    N, K, has_bias, has_res, act, outk = GEMM_KINDS[kind]
    x3 = prec == "fp16x3"
    g = torch.Generator().manual_seed(sum(map(ord, kind)) + M)
    a32 = torch.randn(M, K, generator=g)
    ahi, alo = pair(a32)
    a = (torch.cat([ahi, alo], 1) if x3 else ahi).contiguous().to(dev)
    aref = ahi.double() + alo.double() if x3 else ahi.double()
    w, wref, bias = gemm_weights(kind, prec)
    w = w.to(dev)
    bias_d = bias.to(dev) if bias is not None else None
    res = torch.randn(M, N, generator=g).to(dev) if has_res else None
    split = x3 and outk == "f16"
    if outk == "logits":
        buf = torch.full((M + 1, (N + 7) // 8 * 8), SENTINEL, device=dev)
        out = buf[:M, :N]
    elif outk == "f32":
        buf = torch.full((M + 1, N), SENTINEL, device=dev)
        out = buf[:M]
    else:
        buf = torch.full((M + 1, (2 if split else 1) * N), SENTINEL, dtype=torch.float16, device=dev)
        out = buf[:M]
    _covers(a, a.data_ptr(), M * a.shape[1])
    _covers(w, w.data_ptr(), N * (2 if x3 else 1) * K)
    _covers(buf, out.data_ptr(), (M - 1) * out.stride(0) + (2 if split else 1) * N)
    ops.gemm(a, a.stride(0), w, M, N, K, out, out.stride(0), bias_d, res, res.stride(0) if res is not None else 0, act,
             out_f32=(out.dtype == torch.float32), split=split, x3=x3)
    return buf, (aref, wref, bias, res.cpu() if res is not None else None)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,prec,M", GEMM_CASES)
def test_decode_step_gemm(kind, prec, M):
    N, K, _, _, act, outk = GEMM_KINDS[kind]
    x3 = prec == "fp16x3"
    buf, (aref, wref, bias, res) = issue_gemm(kind, prec, M, DEV)
    torch.cuda.synchronize()
    if x3:                              # fp64 on the exact pair values
        z = aref @ wref.t()
        z = z + bias.double() if bias is not None else z
        z = F.gelu(z) if act == ops.ACT_GELU else z
        ref, rel = (z + res.double() if res is not None else z), TOL_X3
    else:                               # fp32 on the rounded operands
        z = aref.float() @ wref.float().t()
        z = z + bias if bias is not None else z
        z = F.gelu(z) if act == ops.ACT_GELU else z
        ref, rel = (z + res if res is not None else z).double(), TOL_GEMM16
    b = buf.cpu()
    split = x3 and outk == "f16"
    got = _act_value(b[:M], N, split) if outk == "f16" else b[:M, :N].double()
    err, tol = (got - ref).abs().max().item(), _tol(ref, rel)
    assert err < tol, f"max abs err {err:.3g} > {tol:.3g}"
    if split:
        check_canonical(b[:M, :N], b[:M, N:])
    assert bool((b[M] == SENTINEL).all()), "guard row written"
    if outk == "logits":
        assert bool((b[:M, N:] == SENTINEL).all()), "pitch padding written"


# ================================================================================================ CPU: the long-n-gram case
def test_long_ngram_case_needs_more_than_64_bans():
    """The single-call and loop cases for long generations only mean something if HF bans more than 64 ids there and a
    list capped at 64 entries would pick differently."""
    V = 51290
    ids, fin, lg, p = pick_case("long_ngram", V)
    nxt, _, proc = hf_pick(ids, lg, fin, p)
    capped, n_bans = capped_pick(ids, lg, p)
    assert n_bans == 70 and int(torch.isinf(proc[0]).sum()) == 70
    assert int(nxt[0]) == 40000 and capped == 169
    ids, fin, lg, p = pick_case("long_ngram1", V)
    nxt, _, _ = hf_pick(ids, lg, fin, p)
    capped, n_bans = capped_pick(ids, lg, p)
    assert n_bans == 202 and int(nxt[0]) == 250 and capped != 250
    # the loop: by its last steps the (a, c) prefix has recurred more than 64 times, and a capped list diverges
    T, seed = 250, 250
    pp = PickParams(max_len=T + 1)
    hf_seq = torch.full((LOOP_B, 1), START, dtype=torch.long)
    hf_fin = torch.zeros(LOOP_B, dtype=torch.long)
    diverged, most = False, 0
    for step in range(T):
        lg = loop_logits(hf_seq, step, T, V, seed)
        nxt, hf_fin, _ = hf_pick(hf_seq, lg, hf_fin, pp)
        if step not in (0, T - 1):
            c, n = capped_pick(hf_seq[-1:], lg[-1:], pp)        # row 5 runs to the end
            most = max(most, n)
            diverged |= c != int(nxt[-1])
        hf_seq = torch.cat([hf_seq, nxt[:, None]], 1)
    assert most > 64 and diverged


# ================================================================================================ CPU: plan coverage
def classify(name, a):
    """the features of a recorded call that select different kernel code or addressing"""
    if name == "b2p_gemm":
        _A, lda, _W, M, N, K, _o, ldc, bias, res, ldr, act, flags, _st = a
        return ("gemm", M, N, K, lda, ldc, bias is not None, res is not None, ldr, act, flags)
    if name == "b2p_mha_cached":
        _q, ldq, _k, _v, ldnew, _kc, _vc, tmax, _s, _B, heads, _o, ldo, split, _st = a
        return ("mha_cached", ldq, ldnew, tmax, heads, ldo, split)
    if name == "b2p_mha":
        q, ldq, k, v, ldk, _B, Lq, Lk, heads, _o, ldo, split, _st = a
        kq = k - q if Lq > 1 else None                        # self-attention: k, v are column slices of q's rows
        return ("mha", ldq, ldk, Lq, Lk, heads, ldo, split, kq, v - k)
    if name == "b2p_layernorm":
        _x, ldx, _g, _b, eps, _T, C, o16, ld16, o32, ld32, split, _st = a
        return ("layernorm", C, ldx, o16 is not None and ld16, o32 is not None and ld32, split, round(eps, 9))
    if name == "b2p_decoder_embed":
        _E, _seq, seq_ld, _s, _P, _B, C, _o, _st = a
        return ("decoder_embed", seq_ld, C)
    if name == "b2p_encoder_embed":
        _i, n_img, _E, _p, n_prompt, _P, _B, C, _o, _st = a
        return ("encoder_embed", n_img, n_prompt, C)
    if name == "b2p_projector_prep":
        _x, _pos, _B, HW, C, _o, split, _st = a
        return ("projector_prep", HW, C, split)
    if name == "b2p_greedy_pick":
        lg, ld, V, _B, _seq, _sl, _f, _s, ngram, bos, feos, eos, pad, max_len, dump, nunf, _st = a
        return ("greedy_pick", V % 2, V, ld, lg % 8 == 0, ngram, bos, feos, eos, pad, max_len, dump is not None, nunf is not None)
    return None


KERNELS = {"b2p_mha_cached", "b2p_mha", "b2p_layernorm", "b2p_decoder_embed", "b2p_encoder_embed", "b2p_projector_prep",
           "b2p_greedy_pick"}


def test_cases_cover_every_call_class_of_the_florence_plans(rec):  # noqa: F811
    from omniparser_b200.florence_engine import FlorencePlan, FlorenceWeights
    from standin import florence as FS
    sd = FS.florence_standin(0).state_dict()
    plan = set()
    for prec, size, K in (("fp16x3", 64, 6), ("fp16", 64, 6), ("fp16x3", 768, 2)):
        w = FlorenceWeights(sd, torch.device("cpu"), FS.GEN, prec)
        p = FlorencePlan(w, K, 20, FS.PROMPT_IDS, use_graph=False, size=size)
        rec.calls.clear()
        p.encode()
        n_enc = len(rec.calls)
        p.reset_decode(K)
        p.decode_step()
        p.decode_step(forced=True)
        for i, (n, a) in enumerate(rec.calls):
            if n in KERNELS or (n == "b2p_gemm" and i >= n_enc):
                plan.add(classify(n, a))
        del p, w
    rec.calls.clear()
    # this module's tables, launched the same way (CPU tensors; the recorder runs nothing)
    for scen, layout in PICK_CASES:
        for dump in (False, True):
            issue_pick(scen, layout, dump, "cpu")
    for T in (20, 250):
        for dump in (False, True):
            loop_pick(*loop_buffers(T, dump, "cpu"))
    for tmax, R, split in MHA_CACHED_CASES:
        qkv, kc, vc, step, out = mha_cached_buffers(R, tmax, split, "cpu")
        issue_mha_cached(0, qkv, kc, vc, tmax, step, R, out, split)
    for name, R in MHA_ROWS:
        for split in (False, True):
            issue_mha(name, R, split, "cpu")
    for c in DEC_EMBED_CASES:
        issue_decoder_embed(*c, "cpu")
    for n_img, B in ((5, 6), (577, 2)):
        issue_encoder_embed(n_img, B, "cpu")
    for HW in (4, 576):
        for split in (False, True):
            issue_projector_prep(HW, split, "cpu")
    for C in LN_CS:
        for outs in LN_OUTS:
            for split in (False, True):
                issue_layernorm(C, outs, split, "unit", "cpu")
    for kind, prec, M in GEMM_CASES:
        issue_gemm(kind, prec, M, "cpu")
    have = {classify(n, a) for n, a in rec.calls}
    missing = sorted(map(str, plan - have))
    assert not missing, "call classes of the Florence plans without a case in this module:\n" + "\n".join(missing)
    kinds = {c[0] for c in plan}
    assert kinds == {"gemm", "mha_cached", "mha", "layernorm", "decoder_embed", "encoder_embed", "projector_prep", "greedy_pick"}
    assert sum(c[0] == "gemm" for c in plan) == 6 * 2 + 6 and len(plan) >= 40
