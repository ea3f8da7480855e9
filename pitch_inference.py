#!/usr/bin/env python
"""Drop-in for the reference's pitch/inference.py (same flags): the F0 of one recording by CREPE-full on the H100
(`compute_f0_sing`: 20 ms hop, Viterbi in 512-frame segments, every value twice, mean over 5), written as the `.pit.csv`
the inference command lines read, one line per 10 ms.  The weights are crepe/assets/full.pth, where the reference keeps
them.  The wav is read as `hubert_infer.load_audio` reads it (16 kHz).

--f0 picks another of the reference's extractors, each on the device and written by the same `save_csv_pitch`:
`mouth` is compute_f0_mouth (Praat's autocorrelation pitch, praat_f0.py), `salience` is compute_f0_salience
(libf0's salience tracker, salience_f0.py) and `pyin` is pyin_f0.compute_f0_pyin (libf0's pYIN at a 10 ms hop over
50-1000 Hz, 0 where unvoiced; a wrapper of this project's, no reference command calls pyin).  The default, `sing`, is
the CREPE path above."""
import argparse
import os
import sys

sys.path.append(os.path.dirname(os.path.abspath(__file__)))

MODEL = os.path.join("crepe", "assets", "full.pth")


def require_cuda():
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("this build has no CPU path: a CUDA (sm_90a) device is required")


if __name__ == "__main__":
    parser = argparse.ArgumentParser()
    parser.add_argument("-w", "--wav", help="wav", dest="wav", required=True)
    parser.add_argument("-p", "--pit", help="pit", dest="pit", required=True)  # csv for excel
    parser.add_argument("--f0", choices=("sing", "mouth", "salience", "pyin"), default="sing", help="F0 extractor")
    args = parser.parse_args()
    print(args.wav)
    print(args.pit)
    require_cuda()
    if args.f0 == "sing":
        from whisper_vits_svc_b200 import crepe_infer

        crepe_infer.pred_pit(crepe_infer.load_model(MODEL, "cuda"), args.wav, args.pit)
    else:
        from whisper_vits_svc_b200 import hostio, praat_f0, pyin_f0, salience_f0

        compute = {"mouth": praat_f0.compute_f0_mouth, "salience": salience_f0.compute_f0_salience,
                   "pyin": pyin_f0.compute_f0_pyin}[args.f0]
        hostio.save_csv_pitch(compute(args.wav, "cuda"), args.pit)
