#!/usr/bin/env python
"""Drop-in for the reference's prepare/preprocess_train.py (same paths, same files): every item of
./data_svc/waves-32k whose six feature files exist becomes one line
`wave|spec|pitch|hubert|whisper|speaker` of the training lists.  A missing file is printed in red and its item left
out.  The items are shuffled once with `random.shuffle`; the first 10, sorted, go to ./files/valid.txt and the rest to
./files/train.txt.  Speakers and files are walked in os.listdir order and `random` is called as the reference calls
it, so under the same seed both lists are byte-equal to the reference's."""
import argparse
import os
import random
import sys

IndexBySinger = False   # True: one averaged timbre per singer (data_svc/singer) instead of one per file


def print_error(info):
    print(f"\033[31m File isn't existed: {info}\033[0m")


def training_items(rootPath="./data_svc/waves-32k/"):
    """prepare/preprocess_train.py's walk: the list lines of the items whose files all exist."""
    all_items = []
    for spks in os.listdir(f"./{rootPath}"):
        if not os.path.isdir(f"./{rootPath}/{spks}"):
            continue
        print(f"./{rootPath}/{spks}")
        for file in os.listdir(f"./{rootPath}/{spks}"):
            if not file.endswith(".wav"):
                continue
            file = file[:-4]
            if not IndexBySinger:
                path_spk = f"./data_svc/speaker/{spks}/{file}.spk.npy"
            else:
                path_spk = f"./data_svc/singer/{spks}.spk.npy"
            path_wave = f"./data_svc/waves-32k/{spks}/{file}.wav"
            path_spec = f"./data_svc/specs/{spks}/{file}.pt"
            path_pitch = f"./data_svc/pitch/{spks}/{file}.pit.npy"
            path_hubert = f"./data_svc/hubert/{spks}/{file}.vec.npy"
            path_whisper = f"./data_svc/whisper/{spks}/{file}.ppg.npy"
            has_error = False
            for path in (path_spk, path_wave, path_spec, path_pitch, path_hubert, path_whisper):
                if not os.path.isfile(path):
                    print_error(path)
                    has_error = True
            if not has_error:
                all_items.append(f"{path_wave}|{path_spec}|{path_pitch}|{path_hubert}|{path_whisper}|{path_spk}")
    return all_items


def main(argv=None):
    argparse.ArgumentParser(description=__doc__.split("\n\n")[0]).parse_args(argv)
    os.makedirs("./files/", exist_ok=True)
    all_items = training_items()
    random.shuffle(all_items)
    valids = sorted(all_items[:10])
    trains = all_items[10:]
    with open("./files/valid.txt", "w", encoding="utf-8") as fw:
        for strs in valids:
            print(strs, file=fw)
    with open("./files/train.txt", "w", encoding="utf-8") as fw:
        for strs in trains:
            print(strs, file=fw)
    return 0


if __name__ == "__main__":
    sys.exit(main())
