"""Pin the control flow of UniSE's `Model.validation_step` (QuarkAudio-UniSE/model/model.py:134-160) against the REFERENCE'S OWN CODE.

TEST INFRASTRUCTURE.  Run in the build container only:  python -m oracle.make_golden_unise_validation [--out PATH]

Imports the reference's `model/model.py` with the stub packages of oracle/make_golden_unise.py, builds a `Model` WITHOUT running its
`__init__`, plugs the deterministic stand-ins of oracle/unise_validation_stubs.py (tokenizer, LM) and oracle/unise_stubs.py
(`HFSemanticModel`), captures `log_dict`, and runs the reference's unmodified `validation_step` (including its real `stft_logmel`)
over seeded batches.  Writes the logged (loss, acc), the log_dict keyword arguments and the recorded LM call of each case to
tests/golden/unise_validation_glue.npz (the inputs are re-made from the seed).  tests/test_unise_validation_host.py drives
`unified_audio_b200.unise.Model._validation_step` with the same stand-ins and must reproduce them exactly: which waveform is
tokenized, when the enrollment enters the prefix, the squeeze of the global ids, unequal token and feature lengths.
The npz is written with fixed zip timestamps, so a rerun reproduces the file byte for byte.
"""
import argparse
import json
import os
import zipfile

import numpy as np
import torch

from oracle.make_golden_unise import ROOT, import_reference_model

OUT = os.path.join(ROOT, "tests", "golden", "unise_validation_glue.npz")
SEED = 30


def make_cases():
    """name -> the reference's validation batch (mode, enroll, mix, speech, interf, fs, lengths, names); re-made from the seed"""
    g = torch.Generator().manual_seed(SEED)
    w = lambda B, L: 0.1 * torch.randn(B, L, generator=g)
    fs, names = torch.full((2,), 16000, dtype=torch.long), ["a", "b"]
    lengths = lambda L: torch.full((2,), L, dtype=torch.long)
    cases = {}
    mix, speech = w(2, 16000), w(2, 16000)
    cases["se"] = ("se", None, mix, speech, None, fs, lengths(16000), names)
    cases["se_interf"] = ("se", None, mix, speech, w(2, 16000), fs, lengths(16000), names)       # interf given: still tokenizes speech
    enroll, interf = w(2, 12000), w(2, 16000)
    cases["tse"] = ("tse", enroll, mix, speech, interf, fs, lengths(16000), names)
    cases["rtse"] = ("rtse", enroll, mix, speech, interf, fs, lengths(16000), names)
    cases["tse_no_enroll"] = ("tse", None, mix, speech, interf, fs, lengths(16000), names)
    cases["se_unequal"] = ("se", None, w(2, 16640), w(2, 15000), None, fs, lengths(16640), names)
    return cases


def save_npz(path, arrays):
    """np.savez_compressed's layout with fixed entry timestamps"""
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for k, v in arrays.items():
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            with z.open(info, "w") as f:
                np.lib.format.write_array(f, np.asanyarray(v), allow_pickle=False)


def run():
    from oracle import unise_stubs as st
    from oracle import unise_validation_stubs as vs
    Model, _ = import_reference_model()
    m = Model.__new__(Model)
    torch.nn.Module.__init__(m)
    m.config = {}
    m.stft_conf = dict(hop_length=320, win_length=640, n_fft=640, n_mels=80)
    m.tokenizer = vs.Tokenizer()
    m.dnn = vs.Dnn()
    m.semantic_model = st.HFSemanticModel()
    logged = []
    m.log_dict = lambda values, **kw: logged.append((values, kw))
    out = {}
    for name, batch in make_cases().items():
        del logged[:]
        m.dnn.calls = []
        with torch.no_grad():
            m.validation_step(batch, 0)
        assert len(logged) == 1 and len(m.dnn.calls) == 1, (logged, m.dnn.calls)
        values, kw = logged[0]
        assert sorted(values) == ["valid_acc", "valid_loss"]
        out[f"{name}.valid_loss"] = values["valid_loss"].numpy()
        out[f"{name}.valid_acc"] = values["valid_acc"].numpy()
        out[f"{name}.log_kwargs"] = np.array(json.dumps(kw, sort_keys=True))
        out[f"{name}.call"] = np.array(json.dumps(m.dnn.calls[0], sort_keys=True))
        c = m.dnn.calls[0]
        print(name, f"loss {float(values['valid_loss']):.7f} acc {float(values['valid_acc']):.4f}", kw,
              {k: c[k] for k in ("task", "enroll", "B", "mix_frames", "enroll_frames")}, "semantic length", len(c["semantic_ids"][0]))
    meta = dict(reference="QuarkAudio-UniSE/model/model.py:134-160 (unmodified validation_step, stand-ins "
                          "oracle/unise_validation_stubs.py + oracle/unise_stubs.HFSemanticModel)", seed=SEED, cases=list(make_cases()))
    out["meta"] = np.array(json.dumps(meta))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=OUT)
    args = ap.parse_args()
    save_npz(args.out, run())
    print("wrote", args.out, os.path.getsize(args.out), "bytes")


if __name__ == "__main__":
    main()
