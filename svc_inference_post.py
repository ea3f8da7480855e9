#!/usr/bin/env python
"""Drop-in for the reference's svc_inference_post.py (same flags, same printed lines, same model path): silence the
converted audio wherever the source recording has no speech.

The Silero VAD (./vad/assets/silero_vad.jit, relative to the working directory) runs on the H100
(whisper-vits-svc_b200/vad_infer.py); the file is read as a tensor container, its TorchScript is not run.  Speech
segments come from get_speech_timestamps(threshold=0.2) on the 16 kHz source; the converted audio (read at 32 kHz) is
zeroed outside them and written as float32 at 32000 Hz.

Differences, by design: audio is read with `whisper_infer.load_audio`, i.e. .wav only and scipy's `resample_poly`
instead of librosa's resampler, so files not already at 16 kHz / 32 kHz give slightly different samples than the
reference; a source with no samples has no speech and never reaches the device, so the output is all zeros."""
import argparse
import os
import sys

sys.path.append(os.path.dirname(os.path.abspath(__file__)))
from scipy.io.wavfile import write

from whisper_vits_svc_b200 import vad_infer
from whisper_vits_svc_b200.whisper_infer import load_audio

MODEL = os.path.join("vad/assets", "silero_vad.jit")


if __name__ == "__main__":
    parser = argparse.ArgumentParser()
    parser.add_argument("--ref", type=str, required=True, help="Path of ref audio.")
    parser.add_argument("--svc", type=str, required=True, help="Path of svc audio.")
    parser.add_argument("--out", type=str, required=True, help="Path of out audio.")
    args = parser.parse_args()
    print("svc in wave :", args.ref)
    print("svc out wave :", args.svc)
    print("svc post wave :", args.out)

    if not os.path.isfile(MODEL):
        sys.exit(f"VAD model not found: {MODEL} (relative to {os.getcwd()}); copy the reference's vad/assets/silero_vad.jit there")

    ref_wave = load_audio(args.ref, 16000)
    timestamps = []
    if ref_wave.shape[0] > 0:
        model = vad_infer.load_model(MODEL, "cuda")
        probs = model.speech_probs([ref_wave])[0]
        timestamps = vad_infer.get_speech_timestamps(probs, ref_wave.shape[0], threshold=0.2)
    svc_wave = load_audio(args.svc, 32000)
    write(args.out, 32000, vad_infer.silence_outside_speech(timestamps, ref_wave.shape[0], svc_wave))
