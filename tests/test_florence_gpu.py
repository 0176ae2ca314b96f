"""GPU parity of the Florence-2 engine against the fp32 HF oracle (standin/florence.py), 64x64-crop mode.

Checks, in order of the data flow: image tokens, encoder states, teacher-forced logits at every decode step
(tolerance stated below), processed scores / forced tokens, and the free-running greedy ids (must be identical)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from omniparser_b200.florence_engine import FlorencePlan, FlorenceWeights  # noqa: E402
from standin import florence as FS  # noqa: E402

DEV = "cuda:0"
K = 6
T_NEW = 20


@pytest.fixture(scope="module")
def setup():
    m = FS.florence_standin(0)
    g = torch.Generator().manual_seed(7)
    crops = torch.randint(0, 256, (K, 64, 64, 3), dtype=torch.uint8, generator=g)
    crops[0, 16:48, 16:48] = 255   # a structured crop among the noise ones
    pv = FS.pixel_values_from_u8(crops)
    ids = FS.input_ids_for(K)
    with torch.no_grad():
        seq = m.generate(input_ids=ids, pixel_values=pv, max_new_tokens=T_NEW, num_beams=1, do_sample=False)
        out = m(input_ids=ids, pixel_values=pv, decoder_input_ids=seq[:, :-1])
        img = m.get_image_features(pv).pooler_output
    ws = {p: FlorenceWeights(m.state_dict(), torch.device(DEV), FS.GEN, p) for p in ("fp16x3", "fp16")}
    return m, crops, seq, out, img, ws


# precision -> (image/encoder abs tol, logits max-abs tol, logits rms tol, ids must match)
TOL = {"fp16x3": (1e-3, 1e-3, 2e-4, True), "fp16": (2e-2, 3e-2, 6e-3, False)}


@pytest.mark.parametrize("prec", ["fp16x3", "fp16"])
def test_encoder_and_teacher_forced_logits(setup, prec):
    m, crops, seq, out, img, ws = setup
    w = ws[prec]
    tol_enc, tol_max, tol_rms, strict = TOL[prec]
    plan = FlorencePlan(w, K, T_NEW, FS.PROMPT_IDS, use_graph=False)
    plan.crops.copy_(crops.to(DEV))
    plan.encode()
    torch.cuda.synchronize()
    e_img = (plan.img_feat.view(K, 5, 768).cpu() - img).abs().max().item()
    enc_ref = out.encoder_last_hidden_state
    e_enc = (plan.enc_out32.view(K, 13, 768).cpu() - enc_ref).abs().max().item()
    print(f"[{prec}] image tokens max abs err {e_img:.5f} (|ref| max {img.abs().max():.2f}); encoder states max abs err {e_enc:.5f} "
          f"(|ref| max {enc_ref.abs().max():.2f})")
    assert e_img < tol_enc and e_enc < tol_enc
    plan.reset_decode(K)
    ref_logits = out.logits   # [K, T, V]
    worst, worst_rms = 0.0, 0.0
    dump = torch.empty((K, w.vocab), dtype=torch.float32, device=DEV)
    for t in range(seq.shape[1] - 1):
        plan.decode_step(dump=dump, force_tokens=seq[:, t + 1].to(DEV).int())
        torch.cuda.synchronize()
        got = plan.logits.cpu()
        d = (got - ref_logits[:, t]).abs()
        worst = max(worst, d.max().item())
        worst_rms = max(worst_rms, d.pow(2).mean().sqrt().item())
        # picked token (before forcing) equals the oracle's greedy choice at this step
        proc = dump.cpu()
        if strict:
            assert torch.equal(proc.argmax(-1), seq[:, t + 1]), f"step {t}"
    print(f"[{prec}] teacher-forced logits: max abs err {worst:.6f}, worst-step rms err {worst_rms:.6f}, logits std {ref_logits.std():.3f}")
    # north star: fp32 logits within 1e-3 -> met by the fp16x3 mode; plain fp16 operands drift ~5e-3 (DESIGN.md)
    assert worst < tol_max and worst_rms < tol_rms


@pytest.mark.parametrize("use_graph", [False, True])
def test_free_running_ids_identical(setup, use_graph):
    m, crops, seq, out, img, ws = setup
    w = ws["fp16x3"]
    Kp = 32   # padded plan: rows beyond K are inert
    plan = FlorencePlan(w, Kp, T_NEW, FS.PROMPT_IDS, use_graph=use_graph)
    plan.crops.zero_()
    plan.crops[:K].copy_(crops.to(DEV))
    for rep in range(2):   # second pass replays the captured graphs
        plan.encode()
        plan.reset_decode(K)
        steps = 0
        while steps < T_NEW:
            plan.decode_step()
            steps += 1
            if plan.unfinished() == 0:
                break
        plan.join()
        torch.cuda.synchronize()
        got = plan.seq[:K, :steps + 1].cpu().long()
        print(f"graph={use_graph} rep={rep} steps={steps}\n{got[:2]}")
        assert got.shape == seq.shape and torch.equal(got, seq)


# --------------------------------------------------------------------------------------------------------------------
# 768x768 mode: the reference's CPU branch (ref:util/utils.py:123 -- processor default do_resize=True, 577 image tokens)
# --------------------------------------------------------------------------------------------------------------------
K768 = 2


@pytest.fixture(scope="module")
def setup768(setup):
    from PIL import Image
    m, crops, *_rest, ws = setup
    c64 = crops[:K768]
    big = torch.from_numpy(np.stack([np.asarray(Image.fromarray(a.numpy()).resize((768, 768), Image.Resampling.BICUBIC)) for a in c64]))
    pv = FS.pixel_values_from_u8(big)
    ids = FS.input_ids_for(K768, 577)
    with torch.no_grad():
        seq = m.generate(input_ids=ids, pixel_values=pv, max_new_tokens=8, num_beams=1, do_sample=False)
        out = m(input_ids=ids, pixel_values=pv, decoder_input_ids=seq[:, :-1])
        img = m.get_image_features(pv).pooler_output
    return m, c64, big, seq, out, img, ws


def test_768_mode_encoder_logits_and_ids(setup768):
    m, c64, big, seq, out, img, ws = setup768
    w = ws["fp16x3"]
    plan = FlorencePlan(w, K768, 8, FS.PROMPT_IDS, use_graph=False, size=768)
    assert plan.n_img == 577 and plan.L == 585
    plan.crops.copy_(c64.to(DEV))
    plan.encode()
    torch.cuda.synchronize()
    assert torch.equal(plan.crops_in.cpu(), big), "device bicubic resize != Pillow BICUBIC"
    e_img = (plan.img_feat.view(K768, 577, 768).cpu() - img).abs().max().item()
    e_enc = (plan.enc_out32.view(K768, 585, 768).cpu() - out.encoder_last_hidden_state).abs().max().item()
    print(f"[768] image tokens max abs err {e_img:.5f} (|ref| max {img.abs().max():.2f}); encoder states max abs err {e_enc:.5f} "
          f"(|ref| max {out.encoder_last_hidden_state.abs().max():.2f})")
    # the 64x64 mode's bound.  It was 5e-3 while channel_attn_kernel summed 36864 stage-0 tokens in one fp32 running sum:
    # 2.6e-3 / 8.2e-4 then, 1.3e-4 / 7e-5 with chunk sums added in fp64 (one H100 80GB HBM3, 700 W power limit); the
    # kernel's own bound is tested in tests/test_davit_kernels_gpu.py
    assert e_img < 1e-3 and e_enc < 1e-3
    plan.reset_decode(K768)
    dump = torch.empty((K768, w.vocab), dtype=torch.float32, device=DEV)
    worst = 0.0
    for t in range(seq.shape[1] - 1):
        plan.decode_step(dump=dump, force_tokens=seq[:, t + 1].to(DEV).int())
        torch.cuda.synchronize()
        worst = max(worst, (plan.logits.cpu() - out.logits[:, t]).abs().max().item())
        assert torch.equal(dump.cpu().argmax(-1), seq[:, t + 1]), f"step {t}"
    print(f"[768] teacher-forced logits max abs err {worst:.6f}")
    assert worst < 1e-3


def test_768_mode_model_api(setup768):
    """processor(do_resize=True) -> 768x768 u8 -> generate(); and the device-resize chunked route; both == oracle ids."""
    from omniparser_b200.caption import B200Florence2Model, B200Florence2Processor
    from PIL import Image
    m, c64, big, seq, out, img, ws = setup768
    model = B200Florence2Model(m.state_dict(), DEV, FS.GEN, precision="fp16x3")
    proc = B200Florence2Processor()
    inputs = proc(images=[Image.fromarray(a.numpy()) for a in c64], text=["<CAPTION>"] * K768, return_tensors="pt")
    assert tuple(inputs["pixel_values"].shape[1:3]) == (768, 768)
    ids_a = model.generate(input_ids=inputs["input_ids"], pixel_values=inputs["pixel_values"], max_new_tokens=8, num_beams=1,
                           do_sample=False).cpu()
    ids_b = model.generate_chunked(c64.to(DEV), 8, FS.PROMPT_IDS, from_resized=False).cpu()
    ref = seq[:, :ids_a.shape[1]]
    assert torch.equal(ids_a, ref) and torch.equal(ids_b, ref)
