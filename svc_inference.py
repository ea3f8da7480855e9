#!/usr/bin/env python
"""Drop-in for the reference's svc_inference.py (same flags, same output files:
svc_out.wav float32 @ hp.data.sampling_rate and svc_out_pit.wav int16 in the CWD), with the
device path running in libsvc_b200.so.

Differences, by design (SURVEY.md §8 scope): the reference shells out to its Whisper / HuBERT /
CREPE extractors when --ppg/--vec/--pit are missing (svc_inference.py:138-154).  Here --ppg and
--vec are produced in-process by the H100 Whisper encoder / HuBERT-Soft encoder when their
checkpoints are available (whisper_pretrain/large-v2.pt, hubert_pretrain/hubert-soft-0d54a1f4.pt);
CREPE is out of scope (SURVEY.md §8f-4), so --pit must be given.  --enable-retrieval reads the
reference's faiss IVF-Flat indexes without faiss and runs the search and blend on the device
(whisper-vits-svc_b200/retrieval.py)."""
import argparse
import logging
import os
import sys

sys.path.append(os.path.dirname(os.path.abspath(__file__)))
import numpy as np
import torch
from scipy.io.wavfile import write

from whisper_vits_svc_b200 import hostio, hparams, models, retrieval

logger = logging.getLogger(__name__)


def main(args):
    if args.pit is None:
        raise SystemExit("--pit is required: the CREPE pitch extractor is out of scope of this build "
                         "(use the reference's pitch/inference.py to produce it)")
    if not torch.cuda.is_available():
        raise SystemExit("this build has no CPU path: a CUDA (sm_90a) device is required")
    if args.vec is None:   # svc_inference.py:144-148 of the reference, in-process
        from whisper_vits_svc_b200 import hubert_infer
        args.vec = "svc_tmp.vec.npy"
        print(f"Auto run : H100 hubert-soft encoder -w {args.wave} -v {args.vec}")
        hm = hubert_infer.load_model(os.path.join("hubert_pretrain", "hubert-soft-0d54a1f4.pt"), "cuda")
        hubert_infer.pred_vec(hm, args.wave, args.vec)
        del hm
    if args.ppg is None:
        from whisper_vits_svc_b200 import whisper_infer
        args.ppg = "svc_tmp.ppg.npy"
        print(f"Auto run : H100 whisper encoder -w {args.wave} -p {args.ppg}")
        wm = whisper_infer.load_model(os.path.join("whisper_pretrain", "large-v2.pt"), "cuda")
        whisper_infer.pred_ppg(wm, args.wave, args.ppg, "cuda")
    logging.basicConfig(level=logging.DEBUG if args.debug else logging.INFO)
    device = torch.device("cuda")
    hp = hparams.load_hparams(args.config)
    model = models.SynthesizerInfer(hp.data.filter_length // 2 + 1, hp.data.segment_size // hp.data.hop_length, hp)
    hostio.load_svc_model(args.model, model)
    retr = retrieval.create_retrival(args, hp, device)
    model.eval()
    model.to(device)
    spk = torch.FloatTensor(np.load(args.spk))
    print("pitch shift: ", args.shift)
    ppg, vec, pit = hostio.prepare_features(args.ppg, args.vec, args.pit, args.shift)
    out_audio = hostio.svc_infer(model, spk, pit, ppg, vec, hp, device,
                                 retrieval=None if isinstance(retr, retrieval.DummyRetrieval) else retr)
    write("svc_out.wav", hp.data.sampling_rate, out_audio)


if __name__ == '__main__':
    parser = argparse.ArgumentParser()
    parser.add_argument('--config', type=str, required=True, help="yaml file for config.")
    parser.add_argument('--model', type=str, required=True, help="path of model for evaluation")
    parser.add_argument('--wave', type=str, required=True, help="Path of raw audio.")
    parser.add_argument('--spk', type=str, required=True, help="Path of speaker.")
    parser.add_argument('--ppg', type=str, help="Path of content vector.")
    parser.add_argument('--vec', type=str, help="Path of hubert vector.")
    parser.add_argument('--pit', type=str, help="Path of pitch csv file.")
    parser.add_argument('--shift', type=int, default=0, help="Pitch shift key.")
    parser.add_argument('--enable-retrieval', action="store_true", help="Enable index feature retrieval")
    parser.add_argument('--retrieval-index-prefix', default='')
    parser.add_argument('--retrieval-ratio', type=float, default=.5)
    parser.add_argument('--n-retrieval-vectors', type=int, default=3)
    parser.add_argument('--hubert-index-path', required=False)
    parser.add_argument('--whisper-index-path', required=False)
    parser.add_argument('--debug', action="store_true")
    main(parser.parse_args())
