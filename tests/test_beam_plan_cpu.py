"""CPU dry run of beam-search plans through the argument-checking recorder of test_plan_dryrun_cpu, plus the argument
validation of FlorencePlan / generate()."""
import pytest
import torch

from omniparser_b200.caption import B200Florence2Model, beam_settings
from standin import florence as FS
from test_plan_dryrun_cpu import _check, florence, rec  # noqa: F401  (fixtures)


def _check_beam(name, a):
    """b2p_beam_topk / b2p_beam_update argument checks, restated"""
    if name == "b2p_beam_topk":
        _lg, ld, V, B, nb, _seq, seq_ld, _step, ngram, bos, feos, max_len, _bs, _done, _cs, _ci, _st = a
        assert B >= 0 and 1 <= nb <= 16 and B % nb == 0 and 2 * nb <= V <= ld and ngram >= 0
        assert 2 <= max_len <= 8192 and seq_ld >= max_len and bos < V and feos < V
    elif name == "b2p_beam_update":
        (_cs, _ci, V, K, nb, _seq, seq_ld, _src, tmax, _step, _eos, _pad, max_len, es, _lp, lp_pow, *_rest) = a
        assert K >= 0 and 1 <= nb <= 16 and V >= 2 * nb and 2 <= max_len <= 8192 and seq_ld >= max_len
        assert tmax >= max_len - 1 and nb * max_len <= 16384 and es in (0, 1, 2) and lp_pow
    elif name == "b2p_mha_cached_beam":
        assert a[10] >= 0 and a[9] and a[7] >= 1
    elif name == "b2p_mha_grouped":
        assert a[5] >= 0 and a[9] >= 1
    else:
        _check(name, a)


def _plan(w, K, T, **kw):
    from omniparser_b200.florence_engine import FlorencePlan
    return FlorencePlan(w, K, T, FS.PROMPT_IDS, use_graph=False, size=64, **kw)


@pytest.fixture()
def weights(florence):
    from omniparser_b200.florence_engine import FlorenceWeights
    return FlorenceWeights(florence.state_dict(), torch.device("cpu"), FS.GEN, "fp16x3")


def test_greedy_plan_unchanged(rec, weights):
    p = _plan(weights, 2, 4)
    p.encode()
    n_enc = len(rec.calls)
    p.reset_decode(2)
    p.decode_step()
    names = [c[0] for c in rec.calls[n_enc:]]
    assert len(names) == 71 and names[-2:] == ["b2p_greedy_pick", "b2p_step_advance"]
    assert not any("beam" in n or n == "b2p_mha_grouped" for n in names)


@pytest.mark.parametrize("nb,es,lp", [(3, True, 1.0), (5, False, 0.6), (16, "never", 2.0)])
def test_beam_plan_step(rec, weights, nb, es, lp, monkeypatch):
    import test_plan_dryrun_cpu as D
    monkeypatch.setattr(D, "_check", _check_beam)
    K, T = 2, 4
    p = _plan(weights, K, T, num_beams=nb, early_stopping=es, length_penalty=lp)
    p.encode()
    n_enc = len(rec.calls)
    enc = rec.calls[:n_enc]
    assert all(c[1][5] == K for c in enc if c[0] == "b2p_mha")          # the encoder runs on the K crops
    p.reset_decode(K)
    assert p.bscore.view(K, nb)[:, 0].eq(0).all() and p.bscore.view(K, nb)[:, 1:].eq(-1e9).all()
    p.decode_step()
    calls = rec.calls[n_enc:]
    names = [c[0] for c in calls]
    assert len(names) == 72 and names[-3:] == ["b2p_beam_topk", "b2p_beam_update", "b2p_step_advance"]
    assert names.count("b2p_mha_cached_beam") == 6 and names.count("b2p_mha_grouped") == 6
    assert "b2p_mha_cached" not in names and "b2p_mha" not in names and "b2p_greedy_pick" not in names
    R = K * nb
    lm = calls[-4][1]
    assert lm[3] == R and lm[4] == 51290                                  # the LM head runs on every beam row
    topk, upd = calls[-3][1], calls[-2][1]
    assert topk[3] == R and topk[4] == nb and upd[3] == K and upd[4] == nb
    assert upd[13] == {False: 0, True: 1, "never": 2}[es] and abs(upd[14] - lp) < 1e-6
    grouped = [c[1] for c in calls if c[0] == "b2p_mha_grouped"]
    assert all(g[5] == R and g[7] == p.L and g[9] == nb for g in grouped)
    assert p.lp_pow[3].item() == pytest.approx(float(3 ** lp), rel=1e-7)
    n0 = len(rec.calls)
    p.decode_step(forced=True)                                            # forced steps: no LM head
    forced = [c[0] for c in rec.calls[n0:]]
    assert len(forced) == 71 and forced[-4:] == ["b2p_layernorm", "b2p_beam_topk", "b2p_beam_update", "b2p_step_advance"]


def test_beam_plan_refuses_bad_settings(rec, weights, monkeypatch):
    for nb in (0, 17):
        with pytest.raises(ValueError):
            _plan(weights, 2, 4, num_beams=nb)
    for es in ("sometimes", 1, 0, None):                                  # HF tests `early_stopping is True`: 1 is not True
        with pytest.raises(ValueError):
            _plan(weights, 2, 4, num_beams=3, early_stopping=es)
    monkeypatch.setenv("B2P_DECODE_PARTS", "2")
    with pytest.raises(ValueError):
        _plan(weights, 128, 4, num_beams=3)
    with pytest.raises(ValueError):
        _plan(weights, 2, 2000, num_beams=16)                             # 16 * 2001 > 16384 staged ints


def test_generate_argument_validation():
    model = object.__new__(B200Florence2Model)      # validation happens before any device work
    model.beam_defaults = dict(early_stopping=True, length_penalty=0.5)
    for kw, exc in ((dict(num_beams=0), ValueError), (dict(num_beams=17), ValueError),
                    (dict(num_beams=3, num_return_sequences=4), ValueError), (dict(num_beams=1, num_return_sequences=2), ValueError),
                    (dict(do_sample=True), NotImplementedError), (dict(num_beams=3, early_stopping="x"), ValueError),
                    (dict(num_beams=3, early_stopping=1), ValueError), (dict(num_beams=3, early_stopping=0), ValueError)):
        with pytest.raises(exc):
            model.generate(pixel_values=torch.zeros((1, 64, 64, 3), dtype=torch.uint8), **kw)
    assert beam_settings(3, defaults=model.beam_defaults) == dict(num_beams=3, early_stopping=True, length_penalty=0.5,
                                                                  num_return_sequences=1)
    assert beam_settings(3, early_stopping="never", length_penalty=2, num_return_sequences=3) == dict(
        num_beams=3, early_stopping="never", length_penalty=2.0, num_return_sequences=3)
    assert beam_settings(1, early_stopping=True) == dict(num_beams=1, num_return_sequences=1)


def test_beam_defaults_reader(tmp_path):
    import json
    from omniparser_b200.caption import load_beam_defaults
    (tmp_path / "generation_config.json").write_text(json.dumps(dict(FS.GEN, num_beams=3, early_stopping=True)))
    assert load_beam_defaults(tmp_path) == dict(early_stopping=True)
    (tmp_path / "config.json").write_text(json.dumps(dict(text_config=dict(length_penalty=0.8))))
    assert load_beam_defaults(tmp_path) == dict(early_stopping=True, length_penalty=0.8)


def test_plan_keys_resolve_beam_defaults_like_generate():
    """plan_for / plan_ready / warm_plan without early_stopping / length_penalty address the plan generate() uses"""
    model = object.__new__(B200Florence2Model)
    model.beam_defaults = dict(early_stopping=True, length_penalty=0.5)
    key_plan, bs = model._plan_key(40, 20, FS.PROMPT_IDS, 64, 0, 3, None, None)
    gen = beam_settings(3, defaults=model.beam_defaults)
    key_gen, _ = model._plan_key(40, 20, FS.PROMPT_IDS, 64, 0, 3, gen["early_stopping"], gen["length_penalty"])
    assert key_plan == key_gen and key_plan[-3:] == (3, True, 0.5) and bs == dict(num_beams=3, early_stopping=True, length_penalty=0.5)
    assert model._plan_key(40, 20, FS.PROMPT_IDS, 64, 0, 1, None, None)[0] == (64, 20, tuple(FS.PROMPT_IDS), 64, 0)   # greedy key unchanged
    with pytest.raises(ValueError):
        model._plan_key(40, 20, FS.PROMPT_IDS, 64, 0, 3, 1, None)
