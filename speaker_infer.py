#!/usr/bin/env python
"""Drop-in for the reference's speaker/infer.py (same arguments, same output): the 256-d speaker embedding of one
wav, written as float32 [256] with np.save(..., allow_pickle=False).  The LSTM speaker encoder and its mel front
end run on the H100 (whisper-vits-svc_b200/speaker_infer.py).

Difference, by design: the reference also saves the encoder's state dict to "model_small.pth" in the working
directory after every run (speaker/infer.py:104-108), a leftover that overwrites whatever file has that name.
This script writes only the embedding.  --use_cuda and --eval are accepted and ignored: the encoder always runs
on the GPU in inference mode."""
import argparse
import os
import sys
from argparse import RawTextHelpFormatter

sys.path.append(os.path.dirname(os.path.abspath(__file__)))
import numpy as np

from whisper_vits_svc_b200 import speaker_infer


def main(args):
    model = speaker_infer.load_model(args.model_path, args.config_path, "cuda")
    wav = model.load_wav(args.source)
    embed = model.embed([wav])[0].cpu().numpy().astype(np.float32)
    np.save(args.target, embed, allow_pickle=False)


if __name__ == "__main__":
    parser = argparse.ArgumentParser(description="""Compute embedding vectors for each wav file in a dataset.""",
                                     formatter_class=RawTextHelpFormatter)
    parser.add_argument("model_path", type=str, help="Path to model checkpoint file.")
    parser.add_argument("config_path", type=str, help="Path to model config file.")
    parser.add_argument("-s", "--source", help="input wave", dest="source")
    parser.add_argument("-t", "--target", help="output 256d speaker embeddimg", dest="target")
    parser.add_argument("--use_cuda", type=bool, help="flag to set cuda.", default=True)
    parser.add_argument("--eval", type=bool, help="compute eval.", default=True)
    main(parser.parse_args())
