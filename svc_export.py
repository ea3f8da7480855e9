#!/usr/bin/env python
"""Drop-in for the reference's svc_export.py: the generator of a trainer checkpoint -> ./sovits5.0.pth,
{'model_g': <the 903-key SynthesizerInfer state dict>}, the file every conversion CLI loads.

    python svc_export.py --config configs/base.yaml --checkpoint_path chkpt/sovits5.0/sovits5.0_0100.pt

Only model_g's SynthesizerInfer keys are kept (the trainer's enc_q.*, emb_g.* and speaker_classifier.* entries, the
discriminator and the optimizer states are dropped), as in the reference.  It runs without a GPU.  One visible
difference: a SynthesizerInfer key missing from the checkpoint is printed (`<key> is not in the checkpoint`, by
hostio.load_svc_model) before it is written with its default value; the reference copies the default silently."""
import argparse
import os
import sys

sys.path.append(os.path.dirname(os.path.abspath(__file__)))


def main(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument('-c', '--config', type=str, required=True,
                        help="yaml file for config. will use hp_str from checkpoint if not given.")
    parser.add_argument('-p', '--checkpoint_path', type=str, required=True,
                        help="path of checkpoint pt file for evaluation")
    args = parser.parse_args(argv)
    from whisper_vits_svc_b200 import hostio, hparams, models

    hp = hparams.load_hparams(args.config)
    model = models.SynthesizerInfer(hp.data.filter_length // 2 + 1, hp.data.segment_size // hp.data.hop_length, hp)
    hostio.load_svc_model(args.checkpoint_path, model)
    hostio.save_svc_model(model, "sovits5.0.pth")
    return 0


if __name__ == '__main__':
    sys.exit(main())
