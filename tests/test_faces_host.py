"""The plumbing every face shares, without a GPU: the weight formats of ops.py that the GEMM descriptor reads (conv weights as
tap-major planes, dense weights with K padded to a multiple of 64), and the face base class (prepared state dropped when the
parameters or the device change, reference checkpoints loaded strictly with the keys a face ignores)."""
import pytest
import torch
import torch.nn.functional as F

from unified_audio_b200 import ops
from unified_audio_b200.ops import Planes


def _planes64(p: Planes):
    return p.hi.double() + (p.lo.double() if p.lo is not None else 0.0)


@pytest.mark.parametrize("cin,cout,k,stride,dilation", [(1, 32, 7, 1, 1), (37, 20, 3, 1, 1), (64, 64, 1, 1, 1), (100, 48, 7, 1, 3),
                                                        (70, 16, 4, 2, 1), (24, 40, 16, 8, 1), (130, 8, 3, 1, 9)])
def test_conv_planes_contracted_like_the_gemm_reproduce_conv1d(cin, cout, k, stride, dilation):
    """out[t, co] = sum over taps j and padded channels c of A[t * stride + j * dilation, c] * W[co, j * cpad + c]: with the padding
    columns of A filled with garbage, that contraction of conv_planes' weight is F.conv1d in fp64, and the padding is exactly zero."""
    g = torch.Generator().manual_seed(cin * 1000 + k)
    w = torch.randn(cout, cin, k, generator=g, dtype=torch.float64)
    cpad = (cin + 63) // 64 * 64
    for split in (True, False):
        p = ops.conv_planes(w, split)
        assert p.hi.shape == (cout, k * cpad) and (p.lo is not None) == split
        W = _planes64(p).reshape(cout, k, cpad)
        assert bool((p.hi.reshape(cout, k, cpad)[:, :, cin:] == 0).all())
        assert p.lo is None or bool((p.lo.reshape(cout, k, cpad)[:, :, cin:] == 0).all())
        w_planes = W[:, :, :cin].permute(0, 2, 1)                       # the weight the planes hold, [Cout, Cin, k]
        assert float((w_planes - w).abs().max() / w.abs().max()) < (1e-6 if split else 1e-3)
        T = 40
        x = torch.randn(2, cin, T, generator=g, dtype=torch.float64)
        a = torch.full((2, T, cpad), 1e3, dtype=torch.float64)            # channel-last rows, garbage in the padding channels
        a[:, :, :cin] = x.transpose(1, 2)
        T_out = (T - dilation * (k - 1) - 1) // stride + 1
        rows = torch.arange(T_out)[:, None] * stride + torch.arange(k)[None, :] * dilation      # [T_out, k]
        got = torch.einsum("btjc,ojc->bto", a[:, rows], W)
        want = F.conv1d(x, w_planes, stride=stride, dilation=dilation).transpose(1, 2)
        assert got.shape == want.shape and float((got - want).abs().max() / want.abs().max()) < 1e-12
    # the fp32 rounding may happen before or after the permutation and padding: same bits
    a, b = ops.conv_planes(w), ops.conv_planes(w.float())
    assert torch.equal(a.hi, b.hi) and torch.equal(a.lo, b.lo)


def test_pad_k_planes_pads_exactly():
    g = torch.Generator().manual_seed(2)
    for n, kk, kp in ((5, 37, 64), (48, 128, 128), (3, 130, 192)):
        w = torch.randn(n, kk, generator=g)
        for split in (True, False):
            p, ref = ops.pad_k_planes(w, kp, split), Planes.from_f32(w, split)
            assert p.hi.shape == (n, kp) and torch.equal(p.hi[:, :kk], ref.hi) and bool((p.hi[:, kk:] == 0).all())
            if split:
                assert torch.equal(p.lo[:, :kk], ref.lo) and bool((p.lo[:, kk:] == 0).all())
            else:
                assert p.lo is None
        a, b = ops.pad_k_planes(w.double(), kp), ops.pad_k_planes(w, kp)
        assert torch.equal(a.hi, b.hi) and torch.equal(a.lo, b.lo)


# ----------------------------------------------------------------------------- face base class
def _codec():
    from oracle import weights
    from unified_audio_b200.codec import Codec
    cfg = weights.h2_small()
    m = Codec(cfg["encoder_config"], cfg["decoder_config"], cfg["quantizer_config"], cfg["semantic_encoder_config"],
              cfg["semantic_decoder_config"])
    return m, weights.make_h2_state_dict(cfg, 1), {"semantic_decoder.conv1.conv.weight": torch.zeros(4, 4, 3)}


def _codec_h1():
    from oracle import hcodec1
    from unified_audio_b200.codec_h1 import CodecH1
    c = hcodec1.h1_small()
    return CodecH1(_cfg=c), hcodec1.make_state_dict(c, 1), {"semantic_decoder.conv1.conv.weight": torch.zeros(4, 4, 3)}


def _codec_h15():
    from oracle import hcodec15
    from unified_audio_b200.codec_h15 import CodecH15
    c = hcodec15.h15_shallow()
    m = CodecH15(_cfg={k: v for k, v in c.items() if k != "layer_scale"})
    return m, hcodec15.make_state_dict(c, 1), {"semantic_decoder.conv1.conv.weight": torch.zeros(4, 4, 3)}


def _ssl(kind):
    from oracle import hubert as oh
    from oracle import wav2vec2 as ow
    from unified_audio_b200.ssl import SSLFrontEnd
    c, make = dict(hubert=(oh.hubert_small(), oh.make_state_dict), wavlm=(oh.wavlm_small(), oh.wavlm_make_state_dict),
                   wav2vec2=(ow.wav2vec2_small(), ow.make_state_dict))[kind]
    return SSLFrontEnd(dict(c, kind=kind)), make(c, 1), {"masked_spec_embed": torch.zeros(c["hidden"])}


def _lm():
    from oracle import llama
    from unified_audio_b200.llm import LLM_SFT
    c = llama.lm_small()
    m = LLM_SFT(num_tasks=c["num_tasks"], task_map=c["task_map"], feats_dim=c["feats_dim"], llm_base_config=c["llm_base_config"])
    return m, llama.make_lm_state_dict(c, 1), {"cond_input_layer.weight": torch.zeros(4, 4), "rotary_emb.inv_freq": torch.zeros(32)}


def _bicodec(global_tokens):
    from oracle import bicodec as ob
    from oracle import bicodec_global as og
    from unified_audio_b200.bicodec import BiCodec
    c = og.bicodec_global_small()
    sd = dict(ob.make_state_dict(c, 1))
    if global_tokens:
        sd.update(og.make_speaker_state_dict(c, 1))
    ignored = {"encoder.linear_pre.weight": torch.zeros(2, 2), "mel_transformer.spectrogram.window": torch.zeros(640),
               "quantizer.in_project.bias": torch.zeros(8), "speaker_encoder.speaker_encoder.pool.linear1.weight": torch.zeros(2, 2)}
    if global_tokens:
        ignored["speaker_encoder.speaker_encoder.layer1.bn.num_batches_tracked"] = torch.zeros((), dtype=torch.long)
    else:
        ignored["speaker_encoder.perceiver_sampler.latents"] = torch.zeros(8, 16)
    return BiCodec(c, global_tokens=global_tokens), sd, ignored


FACES = {"Codec": _codec, "CodecH1": _codec_h1, "CodecH15": _codec_h15, "SSLFrontEnd-hubert": lambda: _ssl("hubert"),
         "SSLFrontEnd-wavlm": lambda: _ssl("wavlm"), "SSLFrontEnd-wav2vec2": lambda: _ssl("wav2vec2"), "LLM_SFT": _lm,
         "BiCodec": lambda: _bicodec(False), "BiCodec-global": lambda: _bicodec(True)}
# what each face derives from its parameters besides `_w` and `_ws`; all of it must go when they change
EXTRA_STATE = {"Codec": dict(_engine=None), "LLM_SFT": dict(_gen_state={}, _lane_views=None), "BiCodec": dict(_wg=None),
               "BiCodec-global": dict(_wg=None)}


@pytest.mark.parametrize("face", list(FACES))
def test_face_drops_prepared_state_and_loads_reference_checkpoint(face):
    m, sd, ignored = FACES[face]()
    extra = EXTRA_STATE.get(face, {})

    def plant():                          # stand-ins for prepared weights, workspace, captured graphs, engine handles
        m._w, m._ws = {"w": torch.ones(1)}, {("buf", "x", (1,), torch.float32): torch.ones(1)}
        for k in extra:
            setattr(m, k, {"stale": True})

    def dropped():
        return m._w is None and m._ws == {} and type(m._ws) is dict and all(getattr(m, k) == v for k, v in extra.items())

    assert dropped()
    plant()
    m.to("cpu")
    assert dropped()
    plant()
    m.load_state_dict(dict(sd, **ignored), strict=True)
    assert dropped()
    got = m.state_dict()
    assert set(got) == set(sd) and all(torch.equal(got[k], sd[k].to(got[k].dtype)) for k in sd)
    with pytest.raises(RuntimeError):                  # the ignored keys are not optional parameters: a missing real key still fails
        m.load_state_dict({k: v for i, (k, v) in enumerate(sd.items()) if i}, strict=True)
