#!/usr/bin/env python
"""Score trained checkpoints by the trainer's validation loss, `validation/mel_loss` (vits_extend/validation.py), on
the H100, so that the checkpoint to export can be chosen after training.  The reference has no standalone
counterpart: its trainer computes the number only for its current weights, every eval_interval epochs.

    python svc_validate.py -c configs/base.yaml -p chkpt/sovits5.0/*.pt

-p takes trainer checkpoints (model_g, model_d, optimizers, ...) or exported model_g-only files such as
sovits5.0.pth; only model_g's SynthesizerInfer keys are read.  The validation set (hp.data.validation_files) is read
once, with Python's `random` seeded with --seed for the crops, and every checkpoint sees the same crops and the same
random draws (validation.py), so differences between scores come from the weights alone.  It prints one line per
checkpoint, `<path>\t<mel_loss>` at full precision, then `best: <path>\t<mel_loss>`.  A checkpoint that fails to load
is reported on stderr and skipped, and the exit code is then 1.

With --audio-dir DIR it also writes the audio the trainer logs to TensorBoard: for batches idx < hp.log.num_audio, item
0's real audio as DIR/real_{idx}.wav and each checkpoint's fake audio as DIR/<checkpoint file name>/fake_{idx}.wav,
float32 at hp.data.sampling_rate."""
import argparse
import os
import sys

sys.path.append(os.path.dirname(os.path.abspath(__file__)))
import numpy as np
import torch


def main(argv=None):
    parser = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    parser.add_argument("-c", "--config", type=str, required=True, help="yaml file for config.")
    parser.add_argument("-p", "--checkpoint_path", type=str, nargs="+", required=True,
                        help="checkpoints to score (trainer .pt files or exported model_g files)")
    parser.add_argument("--seed", type=int, default=None, help="seed of the crops and draws (default hp.train.seed)")
    parser.add_argument("--batch", type=int, default=None, help="items per batch (default hp.train.batch_size)")
    parser.add_argument("--audio-dir", type=str, default=None, help="write the logged real and fake audio here")
    args = parser.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("this build has no CPU path: a CUDA (sm_90a) device is required")
    from scipy.io.wavfile import write
    from whisper_vits_svc_b200 import hparams, validation

    hp = hparams.load_hparams(args.config)
    seed = int(hp.train.seed if args.seed is None else args.seed)
    batch = int(hp.train.batch_size if args.batch is None else args.batch)
    if batch < 1:
        raise SystemExit(f"--batch {batch}: need at least 1")
    sr = int(hp.data.sampling_rate)
    device = torch.device("cuda")
    scorer = validation.Scorer(hp, device)
    try:
        vset = validation.load_set(hp, hp.data.validation_files, seed, batch, device)
        on_audio = None
        if args.audio_dir:
            os.makedirs(args.audio_dir, exist_ok=True)
            written = set()

            def on_audio(path, idx, real, fake):
                if idx not in written:
                    write(os.path.join(args.audio_dir, f"real_{idx}.wav"), sr, np.asarray(real, np.float32))
                    written.add(idx)
                d = os.path.join(args.audio_dir, os.path.basename(path))
                os.makedirs(d, exist_ok=True)
                write(os.path.join(d, f"fake_{idx}.wav"), sr, np.asarray(fake, np.float32))

        scores, failed = [], 0

        def on_result(path, loss, err):
            nonlocal failed
            if err is not None:
                failed += 1
                print(f"{path}: cannot load: {err}", file=sys.stderr)
                return
            scores.append((loss, path))
            print(f"{path}\t{loss!r}", flush=True)

        scorer.score_paths(args.checkpoint_path, vset, on_result, on_audio)
    finally:
        scorer.close()
    if scores:
        loss, path = min(scores)
        print(f"best: {path}\t{loss!r}")
    return 1 if failed else 0


if __name__ == "__main__":
    sys.exit(main())
