"""Float64 restatements of the training-loop quantities of lvsr/main.py the tests compare with: AdaptiveClipping
(lvsr/extensions.py:64-91), Patience (:157-234), TrackTheBest (blocks.extensions.training) and the alignment
statistics weights_entropy / weights_penalty (lvsr/expressions.py:14-25)."""
import math

import numpy as np


class AdaptiveClipping(object):
    """after_batch(norm) with the main loop's iterations_done = n after batch n; `threshold` is what the next batch
    clips with (initial_threshold before the first)."""

    def __init__(self, initial_threshold, burnin_period, decay_rate):
        self.initial_threshold, self.burnin_period, self.decay_rate = initial_threshold, burnin_period, decay_rate
        self.mean_gradient_norm = self.mean_gradient_norm2 = 0.0
        self.iterations_done = 0
        self.threshold = initial_threshold

    def after_batch(self, norm):
        self.iterations_done += 1
        d = self.decay_rate
        if norm != 0.0:                 # a zero norm leaves the moments unchanged (the reference raises on log(0))
            g = math.log(norm)
            self.mean_gradient_norm = d * self.mean_gradient_norm + (1 - d) * g
            self.mean_gradient_norm2 = d * self.mean_gradient_norm2 + (1 - d) * g ** 2
        var = self.mean_gradient_norm2 - self.mean_gradient_norm ** 2
        std = max(var, 0.0) ** 0.5 if not math.isnan(var) else float("nan")
        threshold = math.exp(self.mean_gradient_norm + std) if not math.isnan(std) else float("nan")
        confidence = min(self.burnin_period, self.iterations_done) / float(self.burnin_period)
        threshold = confidence * threshold + (1 - confidence) * self.initial_threshold
        self.threshold = min(threshold, 5 * self.initial_threshold)
        return self.threshold


def thresholds_of(norms, initial_threshold, burnin_period, decay_rate):
    """The threshold each batch clips with, given the gradient norms of the batches."""
    clip = AdaptiveClipping(initial_threshold, burnin_period, decay_rate)
    out = []
    for n in norms:
        out.append(clip.threshold)
        clip.after_batch(n)
    return out


def track_the_best(values):
    """Indices at which TrackTheBest (choose_best=min) notifies, for the successive values of a record (None: the
    record is absent from that row)."""
    best, out = None, []
    for i, v in enumerate(values):
        if v is None:
            continue
        if best is None or (v != best and min(v, best) == v):
            best = v
            out.append(i)
    return out


def patience_stop_epoch(best_epochs, min_epochs, patience_factor, max_epochs):
    """The epoch after which Patience(min_epochs, patience_factor) stops, given the epochs whose row carries a
    notification (None: it does not stop within max_epochs)."""
    last_best = 0
    for epoch in range(1, max_epochs + 1):
        if epoch in best_epochs:
            last_best = epoch
        if max(min_epochs, int(patience_factor * last_best + 0.5)) <= epoch:
            return epoch
    return None


def alignment_stats(weights, labels_mask=None):
    """(sum of mask * sum_t w log(w + 1e-7), sum over i >= 1 of mask * sum_t max(C_i - C_{i-1}, 0)) in float64."""
    w = np.asarray(weights, dtype=np.float64)
    m = np.ones(w.shape[:2]) if labels_mask is None else np.asarray(labels_mask, dtype=np.float64)
    entropy = float(((w * np.log(w + 1e-7)).sum(axis=2) * m).sum())
    c = np.cumsum(w, axis=2)
    penalty = float((np.maximum(c[1:] - c[:-1], 0).sum(axis=2) * m[1:]).sum())
    return entropy, penalty
