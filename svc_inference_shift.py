#!/usr/bin/env python
"""Drop-in for the reference's svc_inference_shift.py: one recording converted at every pitch shift from --shift_l to
--shift_r (same flags, same printed lines; outputs ./_svc_out/svc_out_{shift}.wav, float32 @ hp.data.sampling_rate,
and svc_out_pit.wav, int16, in the CWD), to find the key that suits the target singer.

The reference calls its `svc_infer` once per shift, a chain of batch-1 device calls each time.  Here the features are
loaded once and every shift is one job of hostio.BatchEngine(ragged=True): the chunks of all shifts run together in
full ragged device batches, and each shift gets its own random draws, as each reference call does.  svc_out_pit.wav is
the last shift's NSF source, as the reference's loop leaves it, from a pitch2source call of its own.

Differences, by design (DESIGN.md §8): the reference's loop calls `svc_infer` without the `retrieval` argument its
svc_inference.py now takes, so it stops with a TypeError; this runs what it intends, without retrieval.  --pit is
required (CREPE is out of scope); a missing --ppg / --vec is extracted in-process as in svc_inference.py."""
import argparse
import os
import sys

sys.path.append(os.path.dirname(os.path.abspath(__file__)))
import numpy as np
import torch
from scipy.io.wavfile import write

from whisper_vits_svc_b200 import hostio, hparams, models

out_path = "./_svc_out"


def main(args):
    if args.pit is None:
        raise SystemExit("--pit is required: the CREPE pitch extractor is out of scope of this build "
                         "(use the reference's pitch/inference.py to produce it)")
    if not torch.cuda.is_available():
        raise SystemExit("this build has no CPU path: a CUDA (sm_90a) device is required")
    args.ppg, args.vec = hostio.extract_missing_features(args.wave, args.ppg, args.vec)
    device = torch.device("cuda")
    hp = hparams.load_hparams(args.config)
    model = models.SynthesizerInfer(hp.data.filter_length // 2 + 1, hp.data.segment_size // hp.data.hop_length, hp,
                                    precision=3)
    hostio.load_svc_model(args.model, model)
    model.eval()
    model.to(device)
    spk = torch.FloatTensor(np.load(args.spk))
    ppg, vec, _ = hostio.prepare_features(args.ppg, args.vec, args.pit)
    pit = hostio.load_csv_pitch(args.pit)    # the integer pitch: every shift scales it in float64
    print(f"pitch shift: [{args.shift_l}, {args.shift_r}]")

    def jobs():
        for shift in range(args.shift_l, args.shift_r + 1):
            print(shift)
            yield shift, spk, hostio.shift_pitch(pit, shift), ppg, vec

    engine = hostio.BatchEngine(model, hp, device, ragged=True)
    for shift, audio in engine.run(jobs()):
        write(os.path.join(out_path, f"svc_out_{shift}.wav"), hp.data.sampling_rate, audio)
    # svc_inference.py:88-92 in the reference's last call: the source of the last shift's pitch, cut to the frames
    # the features share
    last = hostio.shift_pitch(pit, args.shift_r)[:min(len(pit), ppg.size(0), vec.size(0))]
    with torch.no_grad():
        source = model.pitch2source(last.unsqueeze(0).to(device))
        write("svc_out_pit.wav", hp.data.sampling_rate, model.source2wav(source))


if __name__ == '__main__':
    parser = argparse.ArgumentParser()
    parser.add_argument('--config', type=str, required=True, help="yaml file for config.")
    parser.add_argument('--model', type=str, required=True, help="path of model for evaluation")
    parser.add_argument('--wave', type=str, required=True, help="Path of raw audio.")
    parser.add_argument('--spk', type=str, required=True, help="Path of speaker.")
    parser.add_argument('--ppg', type=str, help="Path of content vector.")
    parser.add_argument('--vec', type=str, help="Path of hubert vector.")
    parser.add_argument('--pit', type=str, help="Path of pitch csv file.")
    parser.add_argument('--shift_l', type=int, default=0, help="Pitch shift key for [shift_l, shift_r]")
    parser.add_argument('--shift_r', type=int, default=0, help="Pitch shift key for [shift_l, shift_r]")
    args = parser.parse_args()

    assert args.shift_l >= -12, f"--shift_l {args.shift_l} is below -12"
    assert args.shift_r >= -12, f"--shift_r {args.shift_r} is below -12"
    assert args.shift_l <= 12, f"--shift_l {args.shift_l} is above 12"
    assert args.shift_r <= 12, f"--shift_r {args.shift_r} is above 12"
    assert args.shift_l <= args.shift_r, f"--shift_l {args.shift_l} is above --shift_r {args.shift_r}"

    os.makedirs(out_path, exist_ok=True)

    main(args)
