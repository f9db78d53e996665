"""PCM16 mono WAV files + transcripts -> the flat .npz of compat/lvsr/datasets/npz.py, with the recipes' fbank_dd
features computed on the GPU: what exp/wsj/write_hdf_dataset.sh does with Kaldi (compute-fbank-feats --use-energy
--num-mel-bins=40 | add-deltas; global CMVN stats of the train part applied to every part), without Kaldi.

    python tools/featurize.py --part train=train.lst --part valid=valid.lst --out data.npz [--dither 1.0]

A list has one utterance per line: `<uttid> <wav path> <transcript...>`, the path relative to the list's directory
unless absolute.  Transcripts become one label per character, in the order of the sorted characters of every part
(or --characters); the last label is the end of sentence.  The npz also holds the CMVN stats as `cmvn` [2, D+1].
"""
import argparse
import os
import sys
import wave

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

EOS = "</s>"


def read_list(path):
    base = os.path.dirname(os.path.abspath(path))
    out = []
    with open(path) as f:
        for line in f:
            if not line.strip():
                continue
            parts = line.rstrip("\n").split(None, 2)
            if len(parts) < 2:
                raise ValueError("%s: '<uttid> <wav path> <transcript>' expected, got %r" % (path, line))
            uttid, wav = parts[0], parts[1]
            out.append((uttid, wav if os.path.isabs(wav) else os.path.join(base, wav), parts[2] if len(parts) > 2 else ""))
    return out


def read_wav(path, sample_frequency):
    with wave.open(path, "rb") as w:
        if w.getnchannels() != 1 or w.getsampwidth() != 2 or w.getcomptype() != "NONE":
            raise ValueError("%s: PCM16 mono expected (%d channels, %d bytes per sample, %s)" %
                             (path, w.getnchannels(), w.getsampwidth(), w.getcomptype()))
        if w.getframerate() != int(sample_frequency):
            raise ValueError("%s: %d Hz, the front end expects %d Hz (no resampling)" %
                             (path, w.getframerate(), int(sample_frequency)))
        return np.frombuffer(w.readframes(w.getnframes()), dtype="<i2").astype(np.int16)


def batches(items, waves, fb, batch_size):
    for s in range(0, len(items), batch_size):
        chunk = list(range(s, min(len(items), s + batch_size)))
        for i in chunk:
            if fb.num_frames(len(waves[i])) < 1:
                raise ValueError("utterance %s: %d samples, shorter than one frame" % (items[i][0], len(waves[i])))
        yield chunk


def featurize(parts, out, options, characters=None, batch_size=64, train_part="train"):
    """parts: {part: list file}.  Writes `out`; returns the dict of arrays written."""
    pkg = __import__("__graft_entry__").load_package()
    fb = pkg.Fbank(options)
    items = {p: read_list(f) for p, f in parts.items()}
    if train_part not in items:
        raise ValueError("the CMVN stats come from the %r part, which is not given" % train_part)
    waves = {p: [read_wav(w, options.sample_frequency) for _, w, _ in its] for p, its in items.items()}
    chars = list(characters) if characters else sorted({c for its in items.values() for _, _, t in its for c in t})
    index = {c: i for i, c in enumerate(chars)}
    cmvn = pkg.GlobalCmvn(fb)
    for chunk in batches(items[train_part], waves[train_part], fb, batch_size):
        feats, mask = fb.compute([waves[train_part][i] for i in chunk])
        cmvn.accumulate(feats, mask)
    arrays = dict(num_labels=np.int64(len(chars) + 1), characters=np.array(chars + [EOS]), cmvn=cmvn.stats)
    for p, its in items.items():
        rows = []
        for chunk in batches(its, waves[p], fb, batch_size):
            feats, mask = fb.compute([waves[p][i] for i in chunk], cmvn=cmvn)
            feats = feats.cpu().numpy()
            for j, i in enumerate(chunk):
                rows.append(feats[:fb.num_frames(len(waves[p][i])), j])
        for uttid, _, text in its:
            unknown = set(text) - set(index)
            if unknown:
                raise ValueError("utterance %s: characters %s not in the character set" % (uttid, sorted(unknown)))
        labels = [np.array([index[c] for c in t], np.int64) for _, _, t in its]
        arrays[p + "_features"] = np.concatenate(rows).astype(np.float32)
        arrays[p + "_feature_offsets"] = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
        arrays[p + "_labels"] = np.concatenate(labels + [np.zeros(0, np.int64)])
        arrays[p + "_label_offsets"] = np.concatenate([[0], np.cumsum([len(l) for l in labels])]).astype(np.int64)
        arrays[p + "_uttids"] = np.array([u for u, _, _ in its])
    np.savez(out, **arrays)
    return arrays


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--part", action="append", required=True, metavar="NAME=LIST", help="a part and its list file")
    ap.add_argument("--out", required=True)
    ap.add_argument("--train-part", default="train", help="the part whose CMVN stats every part is normalised with")
    ap.add_argument("--characters", default=None, help="the character set, in label order (default: sorted)")
    ap.add_argument("--batch-size", type=int, default=64)
    ap.add_argument("--sample-frequency", type=float, default=16000.0)
    ap.add_argument("--num-mel-bins", type=int, default=40)
    ap.add_argument("--dither", type=float, default=1.0)
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args(argv)
    pkg = __import__("__graft_entry__").load_package()
    parts = dict(p.split("=", 1) for p in args.part)
    opts = pkg.FbankOptions(sample_frequency=args.sample_frequency, num_mel_bins=args.num_mel_bins, dither=args.dither,
                            seed=args.seed)
    arrays = featurize(parts, args.out, opts, args.characters, args.batch_size, args.train_part)
    for p in parts:
        print("%s: %d utterances, %d frames of %d features" % (p, len(arrays[p + "_uttids"]),
                                                                 len(arrays[p + "_features"]),
                                                                 arrays[p + "_features"].shape[1]))
    print("wrote", args.out)


if __name__ == "__main__":
    main()
