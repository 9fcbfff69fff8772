"""UniSE's validation loss (unified_audio_b200.unise.Model.validation_step / validation_epoch, U/model/model.py:134-160) on the GPU
against the chain of oracles: tokens pinned against the reference's own `BiCodecTokenizer.tokenize`
(tests/golden/bicodec_semantic_small.npz, end-to-end case), WavLM features against oracle/hubert.py, (loss, acc) against
oracle/llama.py's `sft_forward` in fp64.  Small widths first, then the shipped widths at B = 2 x 5 s."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
TOL = 1e-3                       # the LM's own tests use the same bound
MARGIN = 1e-4                    # an oracle arg-max closer than this to the runner-up is a numerically unsafe decision
SEG = 5 * 16000
WAVLM_SMALL = dict(conv_dim=[64] * 7, conv_kernel=[10, 3, 3, 3, 3, 2, 2], conv_stride=[5, 2, 2, 2, 2, 2, 2], hidden=128, layers=2,
                   heads=2, ffn=256, pos_k=16, pos_groups=4, eps=1e-5, num_buckets=32, max_distance=80)


def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / b.abs().max())


def capture_lm_inputs(model):
    """the keyword arguments validation_step hands to the LM, recorded by a forward pre-hook"""
    seen = []
    model.dnn.register_forward_pre_hook(lambda mod, args, kwargs: seen.append(dict(kwargs)), with_kwargs=True)
    return seen


def build_small():
    from oracle import hubert as oh
    from oracle import llama
    from oracle import wav2vec2 as ow
    from oracle.make_golden_bicodec_semantic import e2e_wav2vec2_config, small_config, small_state_dict
    from unified_audio_b200.bicodec import BiCodec
    from unified_audio_b200.llm import LLM_SFT
    from unified_audio_b200.ssl import SSLFrontEnd
    from unified_audio_b200.unise import BiCodecTokenizer, Model
    z = np.load(os.path.join(GOLD, "bicodec_semantic_small.npz"))
    meta = json.loads(str(z["meta"]))
    cfg = small_config()
    codec = BiCodec(cfg, global_tokens=True, semantic_tokens=True)
    codec.load_state_dict(small_state_dict(cfg, meta["seed"]), strict=True)
    wc = e2e_wav2vec2_config()
    w2v = SSLFrontEnd(dict(wc, kind="wav2vec2", do_normalize=True), in_rate=16000)
    w2v.load_state_dict(ow.make_state_dict(wc, meta["w2v_seed"]), strict=True)
    wsd = oh.wavlm_make_state_dict(WAVLM_SMALL, 8)
    wavlm = SSLFrontEnd(dict(WAVLM_SMALL, kind="wavlm"), in_rate=16000, compress=False)
    wavlm.load_state_dict(wsd, strict=True)
    lcfg = llama.lm_small(gsize=4096, ssize=256, feats=WAVLM_SMALL["hidden"])
    lsd = llama.make_lm_state_dict(lcfg, 3, 2.0)
    lm = LLM_SFT(num_tasks=lcfg["num_tasks"], task_map=lcfg["task_map"], feats_dim=lcfg["feats_dim"], llm_base_config=lcfg["llm_base_config"])
    lm.load_state_dict(lsd, strict=True)
    tok = BiCodecTokenizer(codec.cuda(), ref_segment_length=meta["ref_segment_length"], feature_extractor=w2v.cuda())
    model = Model(None, tokenizer=tok, dnn=lm.cuda(), semantic_model=wavlm.cuda())
    return model, z, dict(wsd=wsd, lcfg=lcfg, lsd=lsd)


def small_batch(mode, wav, seed):
    """the waveform `mode` tokenizes is `wav`; the other clean waveform, the mixture's noise and the enrollment are seeded noise"""
    g = torch.Generator().manual_seed(seed)
    other = 0.1 * torch.randn(wav.shape, generator=g)
    mix = wav + 0.5 * other
    enroll = 0.1 * torch.randn(wav.shape[0], 4800, generator=g) if mode != "se" else None
    speech, interf = (other, wav) if mode == "rtse" else (wav, other)
    B = wav.shape[0]
    return (mode, enroll, mix, speech, interf, torch.full((B,), 16000), torch.full((B,), wav.shape[1]), [f"c{i}" for i in range(B)])


def to_cuda(batch):
    return tuple(x.cuda() if torch.is_tensor(x) else x for x in batch)


def oracle_loss(o, mode, efeats, mfeats, gids, sids):
    """fp64 sft_forward -> (loss, acc, logits [B, Lt, V], top-2 margin [B, Lt], targets [B, Lt])"""
    from oracle import llama
    sd64 = {k: v.double() for k, v in o["lsd"].items()}
    d = lambda t: None if t is None else t.double().cpu()
    loss, acc, logits = llama.sft_forward(sd64, o["lcfg"], mode, d(efeats), d(mfeats), gids.cpu(), sids.cpu(), return_logits=True)
    top = logits.topk(2, -1).values
    b = o["lcfg"]["llm_base_config"]
    goff, soff = 3, 3 + b["global_size"]
    B = gids.shape[0]
    col = lambda v: torch.full((B, 1), v, dtype=torch.long)
    targets = torch.cat([gids.cpu().long() + goff, col(1), sids.cpu().long() + soff, col(2)], 1)
    return float(loss), float(acc), logits, top[..., 0] - top[..., 1], targets


@pytest.mark.parametrize("mode", ["se", "tse", "rtse"])
def test_validation_step_small_vs_oracle_chain(lib, mode):
    from oracle import hubert as oh
    model, z, o = build_small()
    seen = capture_lm_inputs(model)
    batch = small_batch(mode, torch.from_numpy(z["e2e_wav"]), 60)
    out = model.validation_step(to_cuda(batch))
    torch.cuda.synchronize()
    loss, acc = out["valid_loss"], out["valid_acc"]
    assert loss.dtype == acc.dtype == torch.float32 and loss.dim() == acc.dim() == 0 and loss.is_cuda and acc.is_cuda
    kw = seen[-1]
    assert kw["task_name"] == mode and (kw["enroll_mel"] is None) == (mode == "se")
    # the tokens the LM is handed are the reference tokenizer's
    gids, sids = kw["global_ids"], kw["semantic_ids"]
    assert gids.dtype == torch.int32 and sids.dtype == torch.int64
    assert torch.equal(gids.cpu(), torch.from_numpy(z["e2e_global"]).squeeze(1)) and torch.equal(sids.cpu(), torch.from_numpy(z["e2e_semantic"]))
    # WavLM features
    _, enroll, mix = batch[:3]
    mfeats = oh.extract_semantic_features(o["wsd"], WAVLM_SMALL, mix)
    efeats = oh.extract_semantic_features(o["wsd"], WAVLM_SMALL, enroll) if enroll is not None else None
    e_feat = rel(kw["mix_feats"], mfeats)
    if enroll is not None:
        e_feat = max(e_feat, rel(kw["enroll_feats"], efeats))
    assert kw["mix_feats"].shape[1] == mix.shape[1] // 320 and kw["mix_feats"].shape[1] != sids.shape[1]
    # loss against the fp64 oracle on the same tokens and the oracle's features
    w_loss, w_acc, w_logits, margin, targets = oracle_loss(o, mode, efeats, mfeats, gids, sids)
    e_loss = abs(float(loss) - w_loss) / abs(w_loss)
    # per-position arg-max through return_logits=True, where the oracle's decision is safe
    l2, a2, logits = model.dnn(**kw, return_logits=True)
    torch.cuda.synchronize()
    assert torch.equal(l2, loss) and torch.equal(a2, acc)
    got_am, want_am = logits.argmax(-1).cpu(), w_logits.argmax(-1)
    safe = margin >= MARGIN
    assert torch.equal(got_am[safe], want_am[safe]), f"{mode}: arg-max differs where the oracle's margin is >= {MARGIN}"
    n, unsafe = targets.numel(), int((~safe).sum())
    assert abs(float(acc) - float((got_am == targets).double().mean())) <= 1e-6             # acc is the arg-max hit rate
    assert abs(float(acc) - w_acc) <= unsafe / n + 1e-6
    print(f"[validation small {mode}] WavLM feats rel {e_feat:.2e}  loss {float(loss):.6f} vs {w_loss:.6f} (rel {e_loss:.2e})  "
          f"acc {float(acc):.6f} vs {w_acc:.6f}  positions below margin {unsafe}/{n}")
    assert e_feat < TOL and e_loss < TOL


def test_validation_step_small_composition_and_epoch(lib):
    model, z, _ = build_small()
    wav = torch.from_numpy(z["e2e_wav"])
    batch = to_cuda(small_batch("tse", wav, 61))
    mode, enroll, mix, speech = batch[:4]
    out = model.validation_step(batch)
    # bit-identical to the three components called by hand
    g, s = model.tokenizer.tokenize(speech)
    loss, acc = model.dnn(task_name=mode, enroll_mel=model.mel_like(enroll), enroll_feats=model.extract_semantic_features(enroll),
                          mix_mel=model.mel_like(mix), mix_feats=model.extract_semantic_features(mix), global_ids=g.squeeze(1),
                          semantic_ids=s)
    torch.cuda.synchronize()
    assert torch.equal(out["valid_loss"], loss) and torch.equal(out["valid_acc"], acc)
    # a second call does not change the first call's outputs
    first = {k: v.clone() for k, v in out.items()}
    model.validation_step(to_cuda(small_batch("se", wav.flip(1).contiguous(), 62)))
    torch.cuda.synchronize()
    assert all(torch.equal(out[k], first[k]) for k in first)
    # validation_epoch over three host batches = the batch-size-weighted mean of the three steps
    batches = [small_batch("se", wav, 63), small_batch("tse", wav[:1], 64), small_batch("rtse", wav, 65)]
    steps = [(b[2].shape[0], model.validation_step(to_cuda(b))) for b in batches]
    ep = model.validation_epoch(batches)
    n = sum(B for B, _ in steps)
    for k in ("valid_loss", "valid_acc"):
        want = sum(B * float(o[k]) for B, o in steps) / n
        assert abs(ep[k] - want) <= 1e-12 * abs(want), (k, ep[k], want)
    print(f"[validation small epoch] {ep}")


def test_validation_step_refuses_detokenize_only_tokenizer(lib):
    """A Model whose tokenizer can only detokenize (what test_step needs) raises the tokenizer's NotImplementedError."""
    from oracle.make_golden_bicodec_semantic import small_config
    from unified_audio_b200.bicodec import BiCodec
    from unified_audio_b200.unise import BiCodecTokenizer
    model, z, _ = build_small()
    model.tokenizer = BiCodecTokenizer(BiCodec(small_config()).cuda())
    with pytest.raises(NotImplementedError, match="feature_extractor"):
        model.validation_step(to_cuda(small_batch("se", torch.from_numpy(z["e2e_wav"]), 66)))


def test_validation_step_shipped_widths(lib):
    """Seeded XLSR-53, WavLM-base-plus, BiCodec with both token paths and the shipped LM at B = 2 x 5 s.  The loss is checked
    against the fp64 oracle fed the GPU's own tokens: that isolates the LM from token flips near a decision boundary."""
    from oracle import bicodec as ob
    from oracle import bicodec_global as og
    from oracle import bicodec_semantic as osm
    from oracle import hubert as oh
    from oracle import llama
    from oracle import wav2vec2 as ow
    from unified_audio_b200.bicodec import BiCodec
    from unified_audio_b200.llm import LLM_SFT
    from unified_audio_b200.ssl import WAV2VEC2_XLSR53, WAVLM_BASE_PLUS, SSLFrontEnd
    from unified_audio_b200.unise import BiCodecTokenizer, Model
    cfg = dict(og.BICODEC_GLOBAL_FULL, encoder=osm.ENCODER_PARAMS)
    sd = dict(ob.make_state_dict(cfg, 2))
    sd.update(og.make_speaker_state_dict(cfg, 2))
    sd.update(osm.make_semantic_state_dict(cfg, 2))
    codec = BiCodec(cfg, global_tokens=True, semantic_tokens=True)
    codec.load_state_dict(sd, strict=True)
    w2v = SSLFrontEnd(WAV2VEC2_XLSR53, in_rate=16000)
    w2v.load_state_dict(ow.make_state_dict(ow.WAV2VEC2_XLSR53, 5), strict=True)
    wsd = oh.wavlm_make_state_dict(oh.WAVLM_BASE_PLUS, 9)
    wavlm = SSLFrontEnd(WAVLM_BASE_PLUS, in_rate=16000, compress=False)
    wavlm.load_state_dict(wsd, strict=True)
    lcfg = llama.LM_FULL
    lsd = llama.make_lm_state_dict(lcfg, 7, 2.0)
    lm = LLM_SFT(num_tasks=lcfg["num_tasks"], task_map=lcfg["task_map"], feats_dim=lcfg["feats_dim"], llm_base_config=lcfg["llm_base_config"])
    lm.load_state_dict(lsd, strict=True)
    model = Model(None, tokenizer=BiCodecTokenizer(codec.cuda(), feature_extractor=w2v.cuda()), dnn=lm.cuda(),
                  semantic_model=wavlm.cuda())
    seen = capture_lm_inputs(model)
    o = dict(lcfg=lcfg, lsd=lsd)
    g = torch.Generator().manual_seed(70)
    for mode, length in (("se", 535), ("tse", 786)):
        speech = 0.1 * torch.randn(2, SEG, generator=g)
        batch = (mode, 0.1 * torch.randn(2, SEG, generator=g) if mode == "tse" else None, speech + 0.05 * torch.randn(2, SEG, generator=g),
                 speech, None, torch.full((2,), 16000), torch.full((2,), SEG), ["a", "b"])
        glob, sem = model.tokenizer.tokenize(batch[3].cuda())
        out = model.validation_step(to_cuda(batch))
        torch.cuda.synchronize()
        kw = seen[-1]
        assert glob.shape == (2, 1, 32) and sem.shape == (2, 249)
        assert torch.equal(kw["global_ids"], glob.squeeze(1)) and torch.equal(kw["semantic_ids"], sem)
        F_mix = kw["mix_feats"].shape[1]
        F_enr = kw["enroll_feats"].shape[1] + 1 if kw["enroll_mel"] is not None else 0
        assert F_mix == 250 and 1 + F_enr + 1 + F_mix + 1 + 32 + 1 + sem.shape[1] == length          # the LM sequence
        loss, acc = float(out["valid_loss"]), float(out["valid_acc"])
        assert np.isfinite(loss) and np.isfinite(acc)
        mfeats = oh.extract_semantic_features(wsd, oh.WAVLM_BASE_PLUS, batch[2])
        efeats = oh.extract_semantic_features(wsd, oh.WAVLM_BASE_PLUS, batch[1]) if mode == "tse" else None
        e_feat = rel(kw["mix_feats"], mfeats)
        w_loss, w_acc, _, margin, _ = oracle_loss(o, mode, efeats, mfeats, kw["global_ids"], kw["semantic_ids"])
        e_loss = abs(loss - w_loss) / abs(w_loss)
        print(f"[validation shipped {mode}] LM sequence {length}  WavLM feats rel {e_feat:.2e}  loss {loss:.6f} vs {w_loss:.6f} "
              f"(rel {e_loss:.2e})  acc {acc:.6f} vs {w_acc:.6f}  positions below margin {int((margin < MARGIN).sum())}/{margin.numel()}")
        assert e_loss < TOL
