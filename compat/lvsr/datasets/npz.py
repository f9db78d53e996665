"""Flat .npz stand-in for H5PYAudioDataset + Data (lvsr/datasets/__init__.py:130-310, lvsr/datasets/h5py.py):

    <part>_features [sum T, F] float32, <part>_feature_offsets [N+1]; <part>_labels [sum L] int64,
    <part>_label_offsets [N+1]; optional <part>_uttids [N]; num_labels; optional characters [num_labels] (str)

`Data` keeps the reference's conventions the engine depends on: eos appended (add_eos, :267-270), batches padded
with masks and transposed to TIME-MAJOR [T,B,F] / [L,B] (:297-309), labels int64."""
import numpy as np


class NpzAudioDataset(object):
    def __init__(self, path, part):
        z = np.load(path, allow_pickle=False)
        self.part = part
        self.features, self.foff = z[part + "_features"], z[part + "_feature_offsets"]
        self.labels, self.loff = z[part + "_labels"], z[part + "_label_offsets"]
        self.uttids = z[part + "_uttids"] if part + "_uttids" in z.files else None
        self.num_labels = int(z["num_labels"])
        self.characters = [str(c) for c in z["characters"]] if "characters" in z.files else None
        self.num_examples = len(self.foff) - 1
        self.num_features = int(self.features.shape[1])
        self.provides_sources = ("recordings", "labels") + (("uttids",) if self.uttids is not None else ())

    def example(self, i):
        ex = dict(recordings=self.features[self.foff[i]:self.foff[i + 1]],
                  labels=self.labels[self.loff[i]:self.loff[i + 1]].astype(np.int64))
        if self.uttids is not None:
            ex["uttids"] = str(self.uttids[i])
        return ex

    def decode(self, labels, keep_eos=False):
        return [self.characters[int(l)] if self.characters else str(int(l)) for l in labels]

    def pretty_print(self, labels, example=None):
        return ("" if self.characters else " ").join(self.decode(labels))


class Data(object):
    def __init__(self, dataset_filename=None, path=None, name_mapping=None, add_eos=True, prepend_eos=False,
                 batch_size=10, validation_batch_size=None, sort_k_batches=None, max_length=None, **unused):
        self.path = path or dataset_filename
        self.name_mapping = name_mapping or {}
        self.add_eos, self.prepend_eos = add_eos, prepend_eos
        self.batch_size, self.sort_k_batches, self.max_length = batch_size, sort_k_batches, max_length
        # lvsr/datasets/__init__.py: the batch size of the validation stream, batch_size when not given
        self.validation_batch_size = validation_batch_size or batch_size
        self.info_dataset = self.get_dataset("train")
        self.num_labels = self.info_dataset.num_labels
        self.num_features = self.info_dataset.num_features
        self.eos_label = self.num_labels - 1 if add_eos else None       # the npz reserves its last symbol for eos
        chars = self.info_dataset.characters        # {character: label}, what the LM's symbol remap reads
        self.character_map = None if chars is None else {c: i for i, c in enumerate(chars)}

    def get_dataset(self, part, add_sources=()):
        return NpzAudioDataset(self.path, self.name_mapping.get(part, part))

    def examples(self, part, shuffle=False, seed=1, num_examples=None):
        ds = self.get_dataset(part)
        order = np.arange(ds.num_examples)
        if shuffle:
            np.random.RandomState(seed).shuffle(order)
        for i in order[:num_examples]:
            ex = ds.example(int(i))
            if self.add_eos:
                ex["labels"] = np.concatenate([ex["labels"], [self.eos_label]]).astype(np.int64)
            if self.max_length and len(ex["recordings"]) > self.max_length:
                continue
            yield ex

    def batches(self, part, shuffle=True, seed=1, batch_size=None):
        """Padded, masked, time-major batches (lvsr/datasets/__init__.py:281-309) of batch_size (default: the data's)
        utterances; sort_k_batches groups utterances of similar length."""
        exs = list(self.examples(part, shuffle=shuffle, seed=seed))
        bs = batch_size or self.batch_size
        k = self.sort_k_batches or 1
        out = []
        for s in range(0, len(exs), bs * k):
            chunk = sorted(exs[s:s + bs * k], key=lambda e: len(e["recordings"]))
            for b in range(0, len(chunk), bs):
                out.append(chunk[b:b + bs])
        for group in out:
            B = len(group)
            T = max(len(e["recordings"]) for e in group)
            L = max(len(e["labels"]) for e in group)
            x = np.zeros((T, B, self.num_features), dtype=np.float32)
            m = np.zeros((T, B), dtype=np.float32)
            y = np.zeros((L, B), dtype=np.int64)
            ym = np.zeros((L, B), dtype=np.float32)
            for j, e in enumerate(group):
                t, l = len(e["recordings"]), len(e["labels"])
                x[:t, j], m[:t, j], y[:l, j], ym[:l, j] = e["recordings"], 1, e["labels"], 1
            yield dict(recordings=x, recordings_mask=m, labels=y, labels_mask=ym)
