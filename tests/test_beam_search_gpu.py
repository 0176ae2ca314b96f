"""Beam search on the GPU against transformers' own beam-search helpers and generate().

1. b2p_beam_topk + b2p_beam_update, driven over whole decodes on crafted logits (no model), against GenerationMixin's
   _get_top_k_continuations / _get_running_beams_for_next_iteration / _update_finished_beams / _check_early_stop_heuristic
   / _beam_search_has_unfinished_sequences fed with HF's processed log-probs.  Every step's logits are drawn so that each
   selection boundary of the crops still open has a margin of at least MARGIN (asserted), far above the ~1e-6 difference
   between the two log_softmax implementations.
2. b2p_mha_cached_beam / b2p_mha_grouped against fp64 and bit for bit against the greedy kernels.
3. generate(num_beams=...) on the seeded stand-in: every returned hypothesis re-scored by HF's fp32 CPU model (processor
   rules, lengths, layout, score within 1e-3), and ids equal to HF's generate() on crops whose selections are decided
   beyond 10x the measured teacher-forced logit error."""
import copy

import pytest
import torch

from omniparser_b200 import ops
from test_decode_step_gpu import D, DEV, HEADS, SENTINEL, TOL_F16, TOL_X3, _act_value, _attn_ref, _same_bits, _tol

pytestmark = pytest.mark.gpu

EOS, PAD, START = 2, 1, 2
NEG = -1.0e9
MARGIN = 1e-3
REAL = -5e8            # scores above this are real; at or below it they carry a -1e9 placeholder term
ES_CODE = {False: 0, True: 1, "never": 2}


def _hf():
    from transformers.generation.utils import GenerationMixin

    class _H(GenerationMixin):
        pass
    return _H()


class HFBeams:
    """HF's beam-search state of K crops, advanced through its own helpers (hf:generation/utils.py:3206-3355)."""

    def __init__(self, K, nb, V, max_len, es, lp, ngram, fb, fe):
        from transformers import (ForcedBOSTokenLogitsProcessor, ForcedEOSTokenLogitsProcessor, LogitsProcessorList,
                                  NoRepeatNGramLogitsProcessor)
        self.H, self.K, self.nb, self.V, self.max_len, self.es, self.lp = _hf(), K, nb, V, max_len, es, lp
        self.rseq = torch.full((K, nb, max_len), PAD, dtype=torch.long)
        self.rseq[:, :, 0] = START
        self.seq = self.rseq.clone()
        self.rscore = torch.zeros(K, nb)
        self.rscore[:, 1:] = NEG
        self.bscore = torch.full((K, nb), NEG)
        self.fin = torch.zeros(K, nb, dtype=torch.bool)
        self.heur = torch.ones(K, 1, dtype=torch.bool)
        self.rbi = torch.full((K, nb, max_len - 1), -1, dtype=torch.int32)
        self.bi = self.rbi.clone()
        self.cur_len = 1
        self.done = torch.zeros(K, dtype=torch.bool)
        procs = [NoRepeatNGramLogitsProcessor(ngram)] if ngram else []
        if fb >= 0:
            procs.append(ForcedBOSTokenLogitsProcessor(fb))
        if fe >= 0:
            procs.append(ForcedEOSTokenLogitsProcessor(max_len, fe))
        self.procs = LogitsProcessorList(procs)

    def processed(self, logits):
        flat = self.rseq[:, :, :self.cur_len].reshape(self.K * self.nb, self.cur_len)
        return self.procs(flat, torch.log_softmax(logits, -1))

    def step(self, logp):
        """one iteration; returns (smallest selection margin among the crops still open, step facts)"""
        H, K, nb, V, cl = self.H, self.K, self.nb, self.V, self.cur_len
        acc = (logp.view(K, nb, V) + self.rscore[:, :, None]).reshape(K, nb * V)
        margin = float("inf")
        srt = acc.sort(-1, descending=True).values[:, :2 * nb + 1]
        top, tseq, tbi = H._get_top_k_continuations(acc, self.rseq, self.rbi, cl, 1, False, 2 * nb, nb, V, K)
        hits = (tseq[:, :, cl] == EOS) | (cl + 1 >= self.max_len)
        self.rseq, self.rscore, self.rbi = H._get_running_beams_for_next_iteration(top, tseq, tbi, hits, nb)
        old_bscore = self.bscore.clone()
        self.seq, self.bscore, self.bi, self.fin = H._update_finished_beams(
            self.seq, tseq, self.bscore, top, self.bi, tbi, self.heur, self.fin, hits, torch.ones(2 * nb, dtype=torch.bool).index_fill_(0, torch.arange(nb, 2 * nb), False),
            nb, cl, 1, self.lp, self.es)
        self.cur_len = cl + 1
        self.heur = H._check_early_stop_heuristic(self.heur, self.rscore, self.bscore, self.fin, self.cur_len, self.max_len, 1,
                                                  self.es, self.lp)
        hl = (self.max_len - 1) if (self.es == "never" and self.lp > 0) else self.cur_len - 1
        best = self.rscore[:, :1] / (hl ** self.lp)
        worst = torch.where(self.fin, self.bscore.min(1, keepdim=True)[0], torch.tensor(NEG))
        facts = dict(eos_top=0, eos_backup=0)
        was_done = self.done.clone()
        for k in range(K):
            if was_done[k]:
                continue
            s = srt[k][srt[k] > REAL]
            if s.numel() > 1:
                margin = min(margin, float((s[:-1] - s[1:]).min()))
            m = torch.cat([old_bscore[k], top[k] / (cl ** self.lp)])
            m = m[m > REAL].sort(descending=True).values[:nb + 1]
            if m.numel() > 1:
                margin = min(margin, float((m[:-1] - m[1:]).min()))
            for s_ in range(nb):
                if self.fin[k, s_] and worst[k, s_] > REAL and best[k, 0] > REAL:
                    margin = min(margin, abs(float(best[k, 0] - worst[k, s_])))
            e = (tseq[k, :, cl] == EOS)
            facts["eos_top"] += int(e[:nb].sum()) * int(cl + 1 < self.max_len)
            facts["eos_backup"] += int(e[nb:].sum()) * int(cl + 1 < self.max_len)
            open_ = H._beam_search_has_unfinished_sequences(self.heur[k:k + 1], self.fin[k:k + 1], hits[k:k + 1], self.es)
            if not bool(open_):
                self.done[k] = True
        return margin, facts


def _logits(g, R, V, t, nb):
    x = 3.0 * torch.randn(R, V, generator=g)
    x[:, 3:6] += 8.0                                    # a few favoured tokens: sequences repeat, n-gram bans fire
    boost = torch.rand(R, generator=g) < 0.3            # EOS near the top of some rows, at every rank
    x[boost, EOS] = x[boost].max(1).values + torch.empty(int(boost.sum())).uniform_(-2.0, 0.5, generator=g)
    return x


def hf_trajectory(case, seed=0):
    """per-step logits [R, V] (margins checked) and HF states after each step, until every crop is done"""
    K, nb, V, T = case["K"], case["nb"], case["V"], case["T"]
    max_len = T + 1
    hf = HFBeams(K, nb, V, max_len, case["es"], case["lp"], case["ngram"], case["fb"], case["fe"])
    steps, done_at = [], [None] * K
    facts = dict(eos_top=0, eos_backup=0, bans_nonzero_beam=0)
    g = torch.Generator().manual_seed(seed)
    for t in range(T):
        for attempt in range(1000):
            logits = _logits(g, K * nb, V, t, nb)
            trial = copy.deepcopy(hf)
            logp = trial.processed(logits)
            m, f = trial.step(logp)
            if m >= MARGIN:
                break
        assert m >= MARGIN, f"step {t}: no logits with selection margin >= {MARGIN} (best {m:.3g})"
        # a token the n-gram processor banned that was among the row's 2 nb best raw logits, on a beam other than 0
        if case["ngram"] and 1 < hf.cur_len < max_len - 1:
            raw = torch.log_softmax(logits, -1)
            top = raw.topk(2 * nb, -1).indices
            banned = torch.isinf(logp) & ~torch.isinf(raw)
            for r in range(K * nb):
                if r % nb and not hf.done[r // nb] and bool(banned[r, top[r]].any()):
                    facts["bans_nonzero_beam"] += 1
        for k_ in f:
            facts[k_] += f[k_]
        hf = trial
        for k in range(K):
            if hf.done[k] and done_at[k] is None:
                done_at[k] = t
        steps.append((logits, copy.deepcopy(hf)))
        if bool(hf.done.all()):
            break
    return steps, done_at, facts


# nb, V / ld, early_stopping, length_penalty, n-gram, forced BOS / EOS, active crops K of Kp, max new tokens T
STEP_CASES = [
    dict(nb=2, V=37, ld=40, es=True, lp=1.0, ngram=3, fb=0, fe=2, K=3, Kp=4, T=14, staggered=True),
    dict(nb=3, V=51290, ld=51296, es=True, lp=1.0, ngram=3, fb=0, fe=2, K=3, Kp=3, T=16, staggered=True),
    dict(nb=3, V=37, ld=40, es=False, lp=0.6, ngram=3, fb=0, fe=2, K=3, Kp=5, T=14, staggered=True),
    dict(nb=5, V=37, ld=40, es="never", lp=2.0, ngram=3, fb=0, fe=2, K=3, Kp=3, T=12),
    dict(nb=5, V=51290, ld=51296, es=False, lp=2.0, ngram=2, fb=-1, fe=-1, K=2, Kp=3, T=12),
    dict(nb=16, V=37, ld=40, es=True, lp=0.6, ngram=3, fb=0, fe=2, K=2, Kp=2, T=10),
    dict(nb=16, V=51290, ld=51296, es="never", lp=1.0, ngram=3, fb=0, fe=2, K=2, Kp=3, T=8),
    dict(nb=4, V=37, ld=40, es=False, lp=1.0, ngram=0, fb=-1, fe=2, K=3, Kp=3, T=10),
]


def _case_id(c):
    return f"nb{c['nb']}-V{c['V']}-es{c['es']}-lp{c['lp']}-ng{c['ngram']}-K{c['K']}of{c['Kp']}"


@pytest.mark.parametrize("case", STEP_CASES, ids=_case_id)
def test_beam_step_kernels_match_hf_helpers(case):
    nb, V, ld, T, K, Kp = case["nb"], case["V"], case["ld"], case["T"], case["K"], case["Kp"]
    max_len, R, Rp = T + 1, K * nb, Kp * nb
    steps, done_at, facts = hf_trajectory(case)
    if case["ngram"] and V < 64:
        assert facts["bans_nonzero_beam"] > 0, "no n-gram ban on a beam other than 0"
    assert facts["eos_top"] > 0 and facts["eos_backup"] > 0, facts
    i32 = dict(dtype=torch.int32, device=DEV)
    logits = torch.full((Rp, ld), float("nan"), device=DEV)
    seq = torch.zeros((Rp, max_len + 1), **i32)
    seq[:, 0] = START
    tmax = max_len
    src = torch.arange(Rp, **i32)[:, None].repeat(1, tmax)
    step = torch.zeros(1, **i32)
    bscore = torch.full((Kp, nb), NEG, device=DEV)
    bscore[:, 0] = 0
    bscore = bscore.view(-1)
    cs, ci = torch.zeros((Rp, 2 * nb), device=DEV), torch.zeros((Rp, 2 * nb), **i32)
    parent = torch.zeros(Rp, **i32)
    hyp_seq = torch.full((Rp, max_len + 1), PAD, **i32)
    hyp_score = torch.full((Rp,), NEG, device=DEV)
    hyp_len, hyp_fin = torch.zeros(Rp, **i32), torch.zeros(Rp, **i32)
    heur, done = torch.ones(Kp, **i32), torch.zeros(Kp, **i32)
    done[K:] = 1                                            # padding crops
    n_open = torch.full((1,), K, **i32)
    lp_pow = torch.tensor([1.0] + [float(L) ** case["lp"] for L in range(1, max_len + 1)], dtype=torch.float32, device=DEV)
    prev_done = torch.zeros(K, dtype=torch.bool)
    for t, (lg, hf) in enumerate(steps):
        forced = (t == 0 and case["fb"] >= 0) or (t == T - 1 and case["fe"] >= 0)
        logits.fill_(float("nan"))
        if not forced:                                      # forced steps must not read the logits
            logits[:R, :V] = lg.to(DEV)
        step.fill_(t)
        ops.beam_topk(logits, ld, V, Rp, nb, seq, seq.stride(0), step, case["ngram"], case["fb"], case["fe"], max_len, bscore, done,
                      cs, ci)
        ops.beam_update(cs, ci, V, Kp, nb, seq, seq.stride(0), src, tmax, step, EOS, PAD, max_len, ES_CODE[case["es"]], case["lp"],
                        lp_pow, bscore, parent, hyp_seq, hyp_score, hyp_len, hyp_fin, heur, done, n_open)
        torch.cuda.synchronize()
        g_done = done.cpu()[:K].bool()
        assert torch.equal(g_done, hf.done), f"step {t}: done {g_done.tolist()}, HF {hf.done.tolist()}"
        assert int(n_open.item()) == int((~hf.done).sum()), f"step {t}: open-crop counter"
        assert bool((done.cpu()[K:] == 1).all())
        cl = t + 1
        g_seq, g_src, g_par, g_bs = seq.cpu(), src.cpu(), parent.cpu(), bscore.cpu()
        for k in range(K):
            if prev_done[k]:
                continue                                    # frozen: HF keeps moving its running beams, which never matter
            for b in range(nb):
                r = k * nb + b
                s = float(hf.rscore[k, b])
                if s <= REAL:
                    continue                                # placeholder beams (ties torch may order otherwise)
                assert int(g_par[r]) == int(hf.rbi[k, b, t]) - k * nb, f"step {t} row {r}: parent"
                assert torch.equal(g_seq[r, :cl + 1].long(), hf.rseq[k, b, :cl + 1]), f"step {t} row {r}: running sequence"
                assert torch.equal(g_src[r, :t + 1], hf.rbi[k, b, :t + 1]), f"step {t} row {r}: cache ancestors"
                assert abs(float(g_bs[r]) - s) <= 1e-5 * max(1.0, abs(s)), f"step {t} row {r}: score {float(g_bs[r])} vs {s}"
        g_hs, g_hsc, g_hl, g_hf = hyp_seq.cpu(), hyp_score.cpu(), hyp_len.cpu(), hyp_fin.cpu()
        for k in range(K):
            for s_ in range(nb):
                r = k * nb + s_
                assert bool(g_hf[r]) == bool(hf.fin[k, s_]), f"step {t} crop {k} slot {s_}: finished flag"
                if not hf.fin[k, s_]:
                    continue
                ref = float(hf.bscore[k, s_])
                assert abs(float(g_hsc[r]) - ref) <= 1e-5 * max(1.0, abs(ref)), f"step {t} crop {k} slot {s_}: score"
                assert torch.equal(g_hs[r, :max_len].long(), hf.seq[k, s_]) and int(g_hs[r, max_len]) == PAD, \
                    f"step {t} crop {k} slot {s_}: hypothesis {g_hs[r].tolist()} vs {hf.seq[k, s_].tolist()}"
                assert int(g_hl[r]) == int((hf.bi[k, s_] >= 0).sum()), f"step {t} crop {k} slot {s_}: length"
        prev_done = hf.done.clone()
    assert bool(prev_done.all())
    if case.get("staggered"):                               # crops that stop at different steps (the others stay frozen)
        assert len(set(done_at)) > 1, f"every crop finished at step {done_at[0]}"


def test_beam_exact_ties_follow_the_documented_rule():
    """exact ties: higher score first, then the lower flat index beam * V + token (Python restatement)"""
    nb, V, ld, max_len = 3, 37, 40, 8
    i32 = dict(dtype=torch.int32, device=DEV)
    lg = torch.zeros(nb, ld, device=DEV)
    lg[:, :V] = torch.tensor([float((v * 7) % 5) for v in range(V)], device=DEV)   # many exactly equal logits in each row
    seq = torch.zeros((nb, max_len + 1), **i32)
    seq[:, 0] = START
    step = torch.ones(1, **i32)                              # cur_len 2: no forcing, no n-gram yet
    bscore = torch.zeros(nb, device=DEV)                     # equal beam scores: ties across beams too
    cs, ci = torch.zeros((nb, 2 * nb), device=DEV), torch.zeros((nb, 2 * nb), **i32)
    ops.beam_topk(lg, ld, V, nb, nb, seq, seq.stride(0), step, 3, -1, -1, max_len, bscore, None, cs, ci)
    torch.cuda.synchronize()
    lp = torch.log_softmax(lg[:, :V].cpu(), -1)
    for b in range(nb):
        order = sorted(range(V), key=lambda v: (-float(lp[b, v]), b * V + v))[:2 * nb]
        assert ci[b].cpu().tolist() == [b * V + v for v in order], f"row {b}"
    src = torch.arange(nb, **i32)[:, None].repeat(1, max_len)
    parent = torch.zeros(nb, **i32)
    hyp_seq = torch.full((nb, max_len + 1), PAD, **i32)
    hyp_score, hyp_len, hyp_fin = torch.full((nb,), NEG, device=DEV), torch.zeros(nb, **i32), torch.zeros(nb, **i32)
    heur, done, n_open = torch.ones(1, **i32), torch.zeros(1, **i32), torch.ones(1, **i32)
    lp_pow = torch.tensor([1.0] + [float(L) for L in range(1, max_len + 1)], device=DEV)
    seq[:, 1] = 5
    ops.beam_update(cs, ci, V, 1, nb, seq, seq.stride(0), src, max_len, step, EOS, PAD, max_len, 1, 1.0, lp_pow, bscore, parent,
                    hyp_seq, hyp_score, hyp_len, hyp_fin, heur, done, n_open)
    torch.cuda.synchronize()
    cand = sorted(((float(lp[b, v]), b * V + v) for b in range(nb) for v in range(V)), key=lambda x: (-x[0], x[1]))[:2 * nb]
    run = [f for s, f in cand if f % V != EOS][:nb]
    assert parent.cpu().tolist() == [f // V for f in run] and seq[:, 2].cpu().tolist() == [f % V for f in run]


# ------------------------------------------------------------------------------------------------ attention kernels
@pytest.mark.parametrize("tmax,nb,K,split", [(21, 3, 2, False), (21, 3, 2, True), (64, 5, 3, True), (33, 16, 1, False)])
def test_mha_cached_beam(tmax, nb, K, split):
    """random ancestor tables against fp64 attention over the logically reordered cache; identity table bit-identical to
    b2p_mha_cached; guard rows / columns untouched"""
    R = K * nb
    g = torch.Generator().manual_seed(tmax + nb + split)
    kc = torch.full((R + 1, tmax, D), SENTINEL, device=DEV)
    kc[:R] = torch.randn(R, tmax, D, generator=g).to(DEV)
    vc = torch.full((R + 1, tmax, D), SENTINEL, device=DEV)
    vc[:R] = torch.randn(R, tmax, D, generator=g).to(DEV)
    qkv = torch.randn(R, 3 * D, generator=g).to(DEV)
    w = 2 if split else 1
    for t in (0, 1, 5, tmax - 1):
        step = torch.full((1,), t, dtype=torch.int32, device=DEV)
        src = (torch.randint(0, nb, (R, tmax), generator=g) + (torch.arange(R) // nb * nb)[:, None]).int()
        out = torch.full((R + 1, w * D + 8), SENTINEL, dtype=torch.float16, device=DEV)
        k2, v2 = kc.clone(), vc.clone()
        ops.mha_cached_beam(qkv, 3 * D, qkv[:, D:], qkv[:, 2 * D:], 3 * D, k2, v2, tmax, step, src.to(DEV), R, HEADS, out,
                            out.stride(0), split=split)
        torch.cuda.synchronize()
        rows = torch.where(torch.arange(t + 1)[None, :] < t, src[:, :t + 1].long(), torch.arange(R)[:, None])
        kn, vn = qkv[:, D:2 * D].cpu(), qkv[:, 2 * D:].cpu()
        k2c, v2c = k2.cpu(), v2.cpu()
        _same_bits(k2c[:R, t], kn, "appended k")
        _same_bits(v2c[:R, t], vn, "appended v")
        Kl = k2c[rows, torch.arange(t + 1)[None, :]]           # [R, t+1, D]
        Vl = v2c[rows, torch.arange(t + 1)[None, :]]
        ref = _attn_ref(qkv[:, :D].cpu().view(R, HEADS, 1, 64), Kl.view(R, t + 1, HEADS, 64).transpose(1, 2),
                        Vl.view(R, t + 1, HEADS, 64).transpose(1, 2)).reshape(R, D)
        o = out.cpu()
        err, tol = (_act_value(o[:R, :w * D], D, split) - ref).abs().max().item(), _tol(ref, TOL_X3 if split else TOL_F16)
        assert err < tol, f"t={t}: max abs err {err:.3g} > {tol:.3g}"
        assert bool((o[R] == SENTINEL).all() and (o[:, w * D:] == SENTINEL).all()), "guard row / columns written"
        assert bool((k2c[R] == SENTINEL).all()), "guard cache row written"
        # identity ancestors: the greedy kernel, bit for bit
        ident = torch.arange(R, dtype=torch.int32, device=DEV)[:, None].repeat(1, tmax)
        o1, o2 = out.clone(), out.clone()
        k3, v3, k4, v4 = kc.clone(), vc.clone(), kc.clone(), vc.clone()
        ops.mha_cached_beam(qkv, 3 * D, qkv[:, D:], qkv[:, 2 * D:], 3 * D, k3, v3, tmax, step, ident, R, HEADS, o1, o1.stride(0), split=split)
        ops.mha_cached(qkv, 3 * D, qkv[:, D:], qkv[:, 2 * D:], 3 * D, k4, v4, tmax, step, R, HEADS, o2, o2.stride(0), split=split)
        torch.cuda.synchronize()
        _same_bits(o1, o2, "identity ancestors vs mha_cached")
        _same_bits(k3, k4, "caches")


@pytest.mark.parametrize("nb,K,Lk,split", [(3, 2, 13, False), (3, 4, 13, True), (5, 2, 585, True), (16, 1, 13, False)])
def test_mha_grouped(nb, K, Lk, split):
    """row r reads crop r / nb's K / V: bit-identical to b2p_mha on K / V replicated per beam"""
    R = K * nb
    g = torch.Generator().manual_seed(nb * 10 + K + Lk)
    q = torch.randn(R, D, generator=g).to(DEV)
    kv = torch.randn(K * Lk, 2 * D, generator=g).to(DEV)
    kv_rep = kv.view(K, 1, Lk, 2 * D).expand(K, nb, Lk, 2 * D).reshape(R * Lk, 2 * D).contiguous()
    w = 2 if split else 1
    o1 = torch.full((R + 1, w * D + 8), SENTINEL, dtype=torch.float16, device=DEV)
    o2 = o1.clone()
    ops.mha_grouped(q, D, kv, kv[:, D:], 2 * D, R, 1, Lk, HEADS, nb, o1, o1.stride(0), split=split)
    ops.mha(q, D, kv_rep, kv_rep[:, D:], 2 * D, R, 1, Lk, HEADS, o2, o2.stride(0), split=split)
    torch.cuda.synchronize()
    _same_bits(o1, o2, "grouped vs replicated")
    assert bool((o1.cpu()[R] == SENTINEL).all() and (o1.cpu()[:, w * D:] == SENTINEL).all())


# ------------------------------------------------------------------------------------------------ end to end
K_E2E = 6
T_E2E = 20


@pytest.fixture(scope="module")
def e2e():
    from standin import florence as FS
    from omniparser_b200.caption import B200Florence2Model
    m = FS.florence_standin(0)
    g = torch.Generator().manual_seed(7)
    crops = torch.randint(0, 256, (K_E2E, 64, 64, 3), dtype=torch.uint8, generator=g)
    crops[0, 16:48, 16:48] = 255
    model = B200Florence2Model(m.state_dict(), DEV, FS.GEN, precision="fp16x3")
    return m, crops, model, FS


def _hf_beam(m, FS, crops, T, **kw):
    with torch.no_grad():
        return m.generate(input_ids=FS.input_ids_for(crops.shape[0], 5 if crops.shape[1] == 64 else 577),
                          pixel_values=FS.pixel_values_from_u8(crops), max_new_tokens=T, do_sample=False,
                          return_dict_in_generate=True, output_scores=True, **kw)


E2E_CASES = [dict(num_beams=3, early_stopping=True), dict(num_beams=4, early_stopping=False, length_penalty=0.6),
             dict(num_beams=3, early_stopping=True, num_return_sequences=3)]
RESCORE_TOL = 1e-3    # |GPU hypothesis score - HF fp32 re-score|


@pytest.fixture(scope="module")
def logit_err(e2e):
    """measured teacher-forced logit error of the fp16x3 decoder: max |logits - HF fp32 logits| over every step of HF's
    best beam-search hypotheses, decoded by the greedy plan with those tokens forced"""
    from omniparser_b200.florence_engine import FlorencePlan
    m, crops, model, FS = e2e
    seq = _hf_beam(m, FS, crops, T_E2E, num_beams=3, early_stopping=True).sequences
    with torch.no_grad():
        out = m(input_ids=FS.input_ids_for(K_E2E), pixel_values=FS.pixel_values_from_u8(crops), decoder_input_ids=seq[:, :-1])
    plan = FlorencePlan(model.weights, K_E2E, T_E2E, FS.PROMPT_IDS, use_graph=False, instance=20)
    plan.crops.copy_(crops.to(DEV))
    plan.encode()
    plan.reset_decode(K_E2E)
    dump = torch.empty((K_E2E, model.weights.vocab), dtype=torch.float32, device=DEV)
    worst = 0.0
    for t in range(seq.shape[1] - 1):
        plan.decode_step(dump=dump, force_tokens=seq[:, t + 1].to(DEV).int())
        torch.cuda.synchronize()
        worst = max(worst, (plan.logits.cpu() - out.logits[:, t]).abs().max().item())
    print(f"measured teacher-forced logit error {worst:.3g}")
    return worst


def _rescore(m, FS, crops_u8, ids, nrs, T, lp, n_img=5):
    """HF fp32 CPU re-score of every returned hypothesis: teacher-forced logits, log_softmax, the checkpoint's processors
    (no-repeat-3-gram, forced BOS, forced EOS at max_length) on the hypothesis' own prefix, summed in fp32 step by step as
    HF accumulates beam scores, / L ** lp.  Also asserts HF's output layout and that no processor rule is broken (every
    chosen token has a finite processed log-prob).  Returns (scores, generated lengths)."""
    from transformers import (ForcedBOSTokenLogitsProcessor, ForcedEOSTokenLogitsProcessor, LogitsProcessorList,
                              NoRepeatNGramLogitsProcessor)
    n, W = ids.shape
    procs = LogitsProcessorList([NoRepeatNGramLogitsProcessor(3), ForcedBOSTokenLogitsProcessor(0),
                                 ForcedEOSTokenLogitsProcessor(T + 1, EOS)])
    with torch.no_grad():
        out = m(input_ids=FS.input_ids_for(n, n_img), pixel_values=FS.pixel_values_from_u8(crops_u8.repeat_interleave(nrs, 0)),
                decoder_input_ids=ids[:, :-1])
    hit = ids[:, 1:] == EOS
    assert bool(hit.any(1).all()), "every hypothesis ends with EOS (forced at max_length)"
    L = hit.float().argmax(1) + 1                                # generated tokens incl. EOS
    assert int(L.max()) == W - 1, "output width is 1 + the longest returned hypothesis"
    for i in range(n):
        assert bool((ids[i, L[i] + 1:] == PAD).all()), f"row {i}: pad after EOS"
    acc = torch.zeros(n)
    for j in range(W - 1):
        lp_j = procs(ids[:, :j + 1], torch.log_softmax(out.logits[:, j].float(), -1))
        v = lp_j.gather(1, ids[:, j + 1:j + 2])[:, 0]
        live = j < L
        assert bool(torch.isfinite(v[live]).all()), f"step {j}: rows {torch.nonzero(live & ~torch.isfinite(v)).flatten().tolist()} pick a token HF's processors forbid"
        acc = torch.where(live, acc + v, acc)
    return torch.stack([acc[i] / (int(L[i]) ** lp) for i in range(n)]), L


def _compare_where_decided(ids, ref, margins, nrs, err, scores=None):
    """ids / scores of the crops whose every HF selection margin exceeds 10x the measured logit error must equal HF's"""
    ok = [k for k, mg in enumerate(margins) if mg > 10 * err]
    print(f"HF selection margins {[f'{m:.1e}' for m in margins]}, 10x logit error {10 * err:.1e}: crops compared {ok}")
    if not ok:
        return
    rows = [k * nrs + j for k in ok for j in range(nrs)]
    w = int((ref.sequences[rows] != PAD).sum(1).max())
    assert torch.equal(ids[rows, :w], ref.sequences[rows, :w])
    if scores is not None:
        assert (scores[rows] - ref.sequences_scores[rows]).abs().max().item() < 1e-3


def _crop_margins(ref, n, T, num_beams, early_stopping, length_penalty=1.0, **_):
    """per crop, the smallest selection margin of HF's own run (replayed from its processed scores) while the crop is open"""
    out = []
    for k in range(n):
        hf = HFBeams(1, num_beams, ref.scores[0].shape[1], T + 1, early_stopping, length_penalty, 3, 0, 2)
        mm = float("inf")
        for sc in ref.scores:
            mg, _ = hf.step(sc[k * num_beams:(k + 1) * num_beams])
            mm = min(mm, mg)
            if bool(hf.done.all()):
                break
        out.append(mm)
    return out


def _check_against_rescore(model, plan, m, FS, crops, ids, nb, nrs, T, lp, n_img=5):
    n = crops.shape[0]
    got = plan.hyp_score.view(plan.K, nb)[:n, :nrs].reshape(-1).cpu()
    got_len = plan.hyp_len.view(plan.K, nb)[:n, :nrs].reshape(-1).cpu()
    assert bool(plan.hyp_fin.view(plan.K, nb)[:n].bool().all().item()), "every hypothesis slot holds a finished sequence"
    assert bool((got.view(n, nrs)[:, :-1] >= got.view(n, nrs)[:, 1:]).all()), "best first within each crop"
    hf_score, L = _rescore(m, FS, crops, ids, nrs, T, lp, n_img)
    assert torch.equal(got_len, L.int()), "hypothesis lengths"
    err = (got - hf_score).abs()
    print(f"re-score: max |GPU - HF fp32| {err.max().item():.3g} over {len(err)} hypotheses")
    assert err.max().item() < RESCORE_TOL, f"rows {torch.nonzero(err >= RESCORE_TOL).flatten().tolist()}: {got} vs {hf_score}"


@pytest.mark.parametrize("kw", E2E_CASES, ids=lambda kw: "-".join(f"{k}{v}" for k, v in kw.items()))
def test_generate_beam_matches_hf(e2e, logit_err, kw):
    """every returned hypothesis re-scored by HF's fp32 model (needs no decided selections); ids / scores equal to HF's
    generate() on the crops whose selections are decided beyond the measured logit error"""
    m, crops, model, FS = e2e
    prompt = torch.tensor([FS.PROMPT_IDS] * K_E2E)          # the processor's input_ids (image tokens are the model's)
    ids = model.generate(input_ids=prompt, pixel_values=crops, max_new_tokens=T_E2E, **kw).cpu()
    nb, nrs, lp = kw["num_beams"], kw.get("num_return_sequences", 1), kw.get("length_penalty", 1.0)
    assert ids.shape[0] == K_E2E * nrs and bool((ids[:, 0] == START).all()) and bool((ids[:, 1] == 0).all())
    plan = model.plan_for(K_E2E, T_E2E, FS.PROMPT_IDS, num_beams=nb, early_stopping=kw["early_stopping"], length_penalty=lp)
    _check_against_rescore(model, plan, m, FS, crops, ids, nb, nrs, T_E2E, lp)
    ref = _hf_beam(m, FS, crops, T_E2E, **kw)
    got = plan.hyp_score.view(plan.K, nb)[:K_E2E, :nrs].reshape(-1).cpu()
    _compare_where_decided(ids, ref, _crop_margins(ref, K_E2E, T_E2E, **kw), nrs, logit_err, got)


def test_generate_beam_graph_eager_and_padded_plans_agree(e2e):
    from omniparser_b200.florence_engine import FlorencePlan
    m, crops, model, FS = e2e
    outs = []
    for inst, (use_graph, Kp) in enumerate(((False, K_E2E), (True, K_E2E), (True, 32))):
        plan = FlorencePlan(model.weights, Kp, T_E2E, FS.PROMPT_IDS, use_graph=use_graph, instance=10 + inst, num_beams=3,
                            early_stopping=True)
        plan.crops.zero_()
        plan.crops[:K_E2E].copy_(crops.to(DEV))
        for rep in range(2):
            outs.append(model.generate_from_device_crops(plan, K_E2E).cpu())
    for o in outs[1:]:
        assert torch.equal(o, outs[0])


def test_generate_beam_768_mode(e2e):
    from PIL import Image
    import numpy as np
    m, crops, model, FS = e2e
    big = torch.from_numpy(np.stack([np.asarray(Image.fromarray(a.numpy()).resize((768, 768), Image.Resampling.BICUBIC))
                                     for a in crops[:2]]))
    ids = model.generate(input_ids=torch.tensor([FS.PROMPT_IDS] * 2), pixel_values=big, max_new_tokens=8, num_beams=3, early_stopping=True).cpu()
    ids_b = model.generate_chunked(crops[:2].to(DEV), 8, FS.PROMPT_IDS, from_resized=False, num_beams=3, early_stopping=True).cpu()
    assert torch.equal(ids, ids_b), "host-resized and device-resized 768 crops"
    plan = model.plan_for(2, 8, FS.PROMPT_IDS, 768, num_beams=3, early_stopping=True)
    _check_against_rescore(model, plan, m, FS, big, ids, 3, 1, 8, 1.0, n_img=577)
