#!/usr/bin/env python
"""Drop-in for the reference's svc_preprocessing.py: the ten data-preparation steps, from ./dataset_raw to the
training lists and the loader check, in the reference's order and with the arguments its command list gives each.

Every step runs its CLI's `main` in this one process, so torch is imported, the CUDA context created and the library
loaded once instead of ten times.  The models are loaded one step at a time and each `main` frees its model before it
returns, so the peak device memory is that of the largest step.  Files that fail inside a step are reported and
skipped by that step; a step that returns non-zero or raises stops the run with status 1, as the reference's loop
stops at the first failing command.  -t is accepted and, as in the reference, not passed on to the steps.

Under torchrun (`python -m torch.distributed.run --nproc-per-node 8 svc_preprocessing.py`) each rank runs the device
steps (1-6 and 8) on its share of the files on cuda:(LOCAL_RANK % device count), and rank 0 alone runs the speaker
average, the file lists and the loader check (7, 9 and 10) once the others are done.  A step that fails on any rank
stops every rank with status 1."""
import argparse
import gc
import importlib
import os
import sys
import traceback

sys.path.append(os.path.dirname(os.path.abspath(__file__)))
import torch

STEPS = [
    "preprocess_a.py -w ./dataset_raw -o ./data_svc/waves-16k -s 16000 -t 0",
    "preprocess_a.py -w ./dataset_raw -o ./data_svc/waves-32k -s 32000 -t 0",
    "preprocess_crepe.py -w data_svc/waves-16k/ -p data_svc/pitch",
    "preprocess_ppg.py -w data_svc/waves-16k/ -p data_svc/whisper",
    "preprocess_hubert.py -w data_svc/waves-16k/ -v data_svc/hubert",
    "preprocess_speaker.py data_svc/waves-16k/ data_svc/speaker -t 0",
    "preprocess_speaker_ave.py data_svc/speaker/ data_svc/singer",
    "preprocess_spec.py -w data_svc/waves-32k/ -s data_svc/specs -t 0",
    "preprocess_train.py",
    "preprocess_zzz.py",
]
# the steps that take the whole data set on the host: under torchrun, rank 0 runs them alone
HOST_STEPS = ("preprocess_speaker_ave.py", "preprocess_train.py", "preprocess_zzz.py")


def step_main(step):
    """(the `main` of a step's CLI, its argument list)."""
    script, *argv = step.split()
    return importlib.import_module(script[:-len(".py")]).main, argv


def run_steps(steps, step_main=step_main):
    """Run `steps` in turn; 0, or 1 at the first step that raises or returns non-zero.  Under torchrun every rank
    runs the device steps on its share of the files, and rank 0 alone runs the host steps while the others wait.
    After each step the ranks agree on its status, so that all of them stop at a failing step and none is left
    waiting for another; they share one gloo group over all the steps."""
    from whisper_vits_svc_b200 import dataset, shard
    rank = shard.env_world()[0]
    with dataset.process_group():
        for step in steps:
            if rank == 0:
                print(f"Command: python {step}", flush=True)
            status = 0
            if rank == 0 or step.split()[0] not in HOST_STEPS:
                try:
                    run, step_argv = step_main(step)   # an import that fails on one rank still joins the agreement
                    status = run(step_argv)
                except (Exception, SystemExit):
                    traceback.print_exc()
                    status = 1
                finally:
                    sys.stdout.flush()
                    gc.collect()
                    torch.cuda.empty_cache()
            if dataset.sum_over_ranks([int(bool(status))])[0]:
                return 1
    return 0


def main(argv=None):
    assert torch.cuda.is_available(), "\033[31m You need GPU to Train! \033[0m"
    from whisper_vits_svc_b200 import shard
    if shard.env_world()[0] == 0:
        print("CPU Count is :", os.cpu_count())
    parser = argparse.ArgumentParser()
    parser.add_argument("-t", type=int, default=0, help="thread count")
    parser.parse_args(argv)
    return run_steps(STEPS)


if __name__ == "__main__":
    sys.exit(main())
