"""Pin oracle/bicodec_forward.py against the reference's own BiCodec and write the golden fixture of BiCodec.forward.

Run in the build container only (reads the reference tree):  python -m oracle.make_golden_bicodec_forward
Builds QuarkAudio-UniSE/model/bicodec's BiCodec through its own constructor with all seven submodules (Encoder, WaveGenerator,
FactorizedVectorQuantize, SpeakerEncoder, the prenet and postnet Decoders, and the mel transformer of `init_mel_transformer`) at
small widths, loads seeded weights and runs the unmodified `BiCodec.forward` in eval mode (bicodec.py:113-149), then the check of
the reference's `__main__` block (bicodec.py:235-257): allclose(forward(batch)["recons"], detokenize(*tokenize(batch))).  The
omegaconf / einx stubs are those of oracle/make_golden_bicodec.py.  The weights of the token paths are those of
tests/golden/bicodec_semantic_small.npz (same seed, the calibrated project_in of tests/golden/bicodec_global_small.npz), the reference
clips are the first three of bicodec_global_small.npz: every FVQ and FSQ decision has a margin well clear of fp32 noise.
Outputs: tests/golden/bicodec_forward_small.npz (inputs and every output of forward), tests/golden/bicodec_postnet_keys.json (the
reference Decoder's keys at POSTNET_PARAMS, under "postnet."), tests/golden/bicodec_forward_pinning_report.json.
"""
import json
import os

import numpy as np
import torch

from oracle.make_golden_bicodec import ROOT, _stub_modules
from oracle.make_golden_bicodec_global import synth_wav

GOLD = os.path.join(ROOT, "tests", "golden")
SEED = 48                  # the semantic fixture's seed: every FVQ margin >= 1e-3, 120 tokens over 256 codes with repeats
FORWARD_SEED, B, T = 7, 3, 40


def small_config():
    from oracle import bicodec_forward as of
    from oracle.make_golden_bicodec_semantic import small_config as semantic_small
    return of.bicodec_forward_small(semantic_small())


def small_state_dict(cfg):
    from oracle import bicodec_forward as of
    from oracle.make_golden_bicodec_semantic import small_state_dict as semantic_sd
    sd = semantic_sd(cfg, SEED)
    sd.update(of.make_forward_state_dict(cfg, FORWARD_SEED))
    return sd


def small_batch(cfg):
    from oracle import bicodec_semantic as osm
    g = np.load(os.path.join(GOLD, "bicodec_global_small.npz"))
    feat = osm.synth_feat(B, T, cfg["encoder"]["input_channels"], SEED + 100)
    return {"feat": feat, "ref_wav": torch.from_numpy(g["ref_wav"][:B]).clone(), "wav": synth_wav(B, T * cfg["hop"], FORWARD_SEED + 300)}


def build_reference(cfg, sd):
    _stub_modules()
    from model.bicodec.bicodec import BiCodec
    from model.bicodec.modules.encoder_decoder.feat_decoder import Decoder
    from model.bicodec.modules.encoder_decoder.feat_encoder import Encoder
    from model.bicodec.modules.encoder_decoder.wave_generator import WaveGenerator
    from model.bicodec.modules.speaker.speaker_encoder import SpeakerEncoder
    from model.bicodec.modules.vq.factorized_vector_quantize import FactorizedVectorQuantize
    q, s = cfg["quantizer"], cfg["speaker"]
    model = BiCodec(mel_params=cfg["mel_params"], encoder=Encoder(**cfg["encoder"]), decoder=WaveGenerator(**cfg["decoder"]),
                    quantizer=FactorizedVectorQuantize(q["input_dim"], q["codebook_size"], q["codebook_dim"], commitment=0.25),
                    speaker_encoder=SpeakerEncoder(input_dim=cfg["mel_params"]["num_mels"], out_dim=s["out_dim"], latent_dim=s["latent_dim"],
                                                   token_num=s["token_num"], fsq_levels=s["fsq_levels"],
                                                   fsq_num_quantizers=s["fsq_num_quantizers"]),
                    prenet=Decoder(**cfg["prenet"]), postnet=Decoder(**cfg["postnet"]))
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert not unexpected, unexpected
    bad = [k for k in missing if not k.startswith(("quantizer.cluster_size", "mel_transformer.")) and not k.endswith("num_batches_tracked")]
    assert not bad, bad
    return model.eval()


def rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).abs().max() / b.abs().max())


def main():
    from oracle import bicodec_forward as of
    from oracle import bicodec_global as og
    from oracle import bicodec_semantic as osm
    report = {}
    cfg = small_config()
    sd = small_state_dict(cfg)
    batch = small_batch(cfg)
    model = build_reference(cfg, sd)
    with torch.no_grad():
        out = model(batch)
        sem, glob = model.tokenize(batch)
        recon = model.detokenize(sem, glob)
    report["reference_self_test"] = dict(allclose=bool(torch.allclose(out["recons"].detach(), recon)),
                                         max_abs_diff=float((out["recons"] - recon).abs().max()), recons_absmax=float(recon.abs().max()))
    print("reference self-test", report["reference_self_test"])
    sd64 = {k: v.double() for k, v in sd.items()}
    b64 = {k: v.double() for k, v in batch.items()}
    taps = {}
    got = of.forward(sd64, cfg, b64, taps)
    assert torch.equal(taps["semantic"], sem) and torch.equal(taps["global_tokens"], glob)
    counts = torch.bincount(sem.reshape(-1), minlength=cfg["quantizer"]["codebook_size"])
    r = {k: rel(got[k], out[k]) for k in ("recons", "pred_feat", "x_vector", "d_vector", "perplexity")}
    r.update(cluster_size_equal=bool(float(out["cluster_size"]) == got["cluster_size"]), cluster_size=float(out["cluster_size"]),
             perplexity_value=float(out["perplexity"]), vq_loss_is_nan=bool(torch.isnan(out["vq_loss"])), tokens=int(sem.numel()),
             repeated_codes=int((counts > 1).sum()), fvq_min_margin=float(osm.fvq_margins(sd64, taps["encoder"]).min()),
             fsq_min_margin=float(og.fsq_margins(og.fsq_tokenize(sd64, cfg, og.perceiver(sd64, cfg, taps["latent"]))[1], cfg["speaker"]["fsq_levels"]).min()),
             dtypes={k: str(out[k].dtype) for k in ("recons", "pred_feat", "x_vector", "d_vector", "perplexity", "cluster_size", "vq_loss")},
             shapes={k: list(out[k].shape) for k in ("recons", "pred_feat", "x_vector", "d_vector", "audios")})
    report["small"] = r
    print("small", r)
    assert max(r[k] for k in ("recons", "pred_feat", "x_vector", "d_vector", "perplexity")) < 1e-5, r
    assert r["cluster_size_equal"] and r["vq_loss_is_nan"] and r["repeated_codes"] > 0 and 1 < r["cluster_size"] < r["tokens"]
    assert r["fvq_min_margin"] >= 1e-3 and r["fsq_min_margin"] >= 1e-3, r
    assert out["with_speaker_loss"] is False and torch.equal(out["audios"], batch["wav"].unsqueeze(1))
    np.savez_compressed(os.path.join(GOLD, "bicodec_forward_small.npz"),
                        meta=json.dumps(dict(seed=SEED, forward_seed=FORWARD_SEED, B=B, T=T, feat_seed=SEED + 100, wav_seed=FORWARD_SEED + 300,
                                             ref_wav="bicodec_global_small.npz ref_wav[:3]")),
                        feat=batch["feat"].numpy(), ref_wav=batch["ref_wav"].numpy(), wav=batch["wav"].numpy(),
                        semantic=sem.numpy(), global_tokens=glob.numpy(),
                        **{k: out[k].detach().numpy() for k in ("recons", "pred_feat", "x_vector", "d_vector", "perplexity", "cluster_size",
                                                                 "vq_loss")})
    # ---- the postnet's reference keys at POSTNET_PARAMS
    from model.bicodec.modules.encoder_decoder.feat_decoder import Decoder
    keys = {"postnet." + k: list(v.shape) for k, v in Decoder(**of.POSTNET_PARAMS).state_dict().items()}
    assert keys == {k: list(v[0]) for k, v in of.forward_param_specs(of.BICODEC_FORWARD_FULL).items() if k.startswith("postnet.")}
    json.dump(keys, open(os.path.join(GOLD, "bicodec_postnet_keys.json"), "w"), indent=0)
    json.dump(report, open(os.path.join(GOLD, "bicodec_forward_pinning_report.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
