"""Filterbank front end on the GPU: the recipes' fbank_dd features (Kaldi's compute-fbank-feats --use-energy
--num-mel-bins=40 | add-deltas | apply-global-cmvn, exp/wsj/write_hdf_dataset.sh:94-105) straight from waveforms.

    fb = Fbank(FbankOptions())                     # Kaldi's option names and defaults, deltas of order 2
    x, m = fb.compute(waves)                       # recordings [T, B, 123], recordings_mask [T, B] on the GPU
    cmvn = GlobalCmvn(fb); cmvn.accumulate(x, m)   # Kaldi's [2, D+1] stats, over as many batches as wanted
    x, m = fb.compute(waves, cmvn=cmvn)            # normalised: what SpeechRecognizer.encode / cost take

The computation is the C ABI's lvsr_frontend_* (include/lvsr_b200.h; definition in DESIGN §1 (j)).
"""
import ctypes as C

import numpy as np

from . import _lib

_DEFAULTS = dict(sample_frequency=16000.0, frame_length=25.0, frame_shift=10.0, dither=1.0, remove_dc_offset=True,
                 preemphasis_coefficient=0.97, window_type="povey", round_to_power_of_two=True, snip_edges=True,
                 num_mel_bins=40, low_freq=20.0, high_freq=0.0, use_energy=True, raw_energy=True, energy_floor=0.0,
                 use_log_fbank=True, use_power=True, htk_compat=False, vtln_warp=1.0, delta_order=2, delta_window=2,
                 seed=1)


class FbankOptions(object):
    """compute-fbank-feats' options under Kaldi's names and defaults, plus add-deltas' delta_order / delta_window and
    the seed of the dither draws.  Validated by lvsr_frontend_create."""

    def __init__(self, **kwargs):
        unknown = set(kwargs) - set(_DEFAULTS)
        if unknown:
            raise TypeError("unknown fbank options: %s" % ", ".join(sorted(unknown)))
        for k, v in _DEFAULTS.items():
            setattr(self, k, kwargs.get(k, v))

    def as_dict(self):
        return {k: getattr(self, k) for k in _DEFAULTS}

    def _struct(self):
        if self.window_type not in _lib.WINDOW_TYPES:
            raise ValueError("window_type %r unsupported (%s)" % (self.window_type, ", ".join(_lib.WINDOW_TYPES)))
        s = _lib.LvsrFbankOptions()
        for name, ctype in _lib.LvsrFbankOptions._fields_:
            v = getattr(self, name)
            setattr(s, name, _lib.WINDOW_TYPES[v] if name == "window_type" else
                    (float(v) if ctype is C.c_double else int(v)))
        return s


def _torch():
    import torch
    if not torch.cuda.is_available():
        raise RuntimeError("the filterbank front end needs a CUDA device (no CPU fallback)")
    return torch


class Fbank(object):
    """One lvsr_frontend handle on `device` (default: the current CUDA device)."""

    def __init__(self, options=None, device=None):
        self.options = options or FbankOptions()
        self._handle = None
        struct = self.options._struct()
        lib = _lib.load()
        torch = _torch()
        self.device = torch.device(device if device is not None else "cuda")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        h = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(lib.lvsr_frontend_create(C.byref(struct), C.byref(h)))
        self._handle = h
        self.feature_dim = lib.lvsr_frontend_feature_dim(h)

    def __del__(self):
        try:
            if self._handle is not None:
                _lib.load().lvsr_frontend_destroy(self._handle)
                self._handle = None
        except Exception:
            pass

    def num_frames(self, num_samples):
        return int(_lib.load().lvsr_frontend_num_frames(self._handle, int(num_samples)))

    def _stream(self):
        return _torch().cuda.current_stream(self.device).cuda_stream

    def _samples(self, waveforms, lengths):
        """-> (float32 [B, stride] on the device, 16-byte aligned, stride a multiple of 4; lengths int64 [B])."""
        torch = _torch()
        if isinstance(waveforms, torch.Tensor) or (isinstance(waveforms, np.ndarray) and waveforms.ndim == 2):
            x = torch.as_tensor(waveforms)
            if x.ndim != 2:
                raise ValueError("waveforms: [B, N] expected, got %s" % (tuple(x.shape),))
            lens = np.full(x.shape[0], x.shape[1], np.int64) if lengths is None else np.asarray(lengths, np.int64)
        else:
            rows = [np.asarray(w) for w in waveforms]
            if any(r.ndim != 1 for r in rows):
                raise ValueError("waveforms: one 1-D array per utterance expected")
            lens = np.array([len(r) for r in rows], np.int64) if lengths is None else np.asarray(lengths, np.int64)
            dtype = np.int16 if all(r.dtype == np.int16 for r in rows) else np.float32
            x = np.zeros((len(rows), max(len(r) for r in rows)), dtype)
            for b, r in enumerate(rows):
                x[b, :len(r)] = r
            x = torch.from_numpy(x)
        if lens.shape != (x.shape[0],):
            raise ValueError("lengths: %d entries expected" % x.shape[0])
        x = x.to(self.device).to(torch.float32)
        pad = -x.shape[1] % 4
        if pad:
            x = torch.nn.functional.pad(x, (0, pad))
        if not x.is_contiguous() or x.data_ptr() % 16:
            x = x.contiguous().clone()
        return x, np.ascontiguousarray(lens)

    def compute(self, waveforms, lengths=None, cmvn=None, T=None):
        """Features of a batch -> (recordings [T, B, D], recordings_mask [T, B]) float32 CUDA tensors, frames past an
        utterance's end exactly 0 with mask 0.  waveforms: a list of 1-D int16 / float arrays in int16 units, or a
        [B, N] array or tensor with `lengths` (default: N each).  T: frames of the output (default: the longest
        utterance's).  cmvn: a GlobalCmvn or [2, D+1] stats to normalise with (None: no CMVN)."""
        torch = _torch()
        x, lens = self._samples(waveforms, lengths)
        B = x.shape[0]
        if T is None:
            T = max(1, max(self.num_frames(n) for n in lens))
        stats = None if cmvn is None else _device_stats(cmvn, self.device, self.feature_dim)
        feats = torch.empty((T, B, self.feature_dim), dtype=torch.float32, device=self.device)
        mask = torch.empty((T, B), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().lvsr_frontend_compute(
                self._handle, x.data_ptr(), x.shape[1], lens.ctypes.data_as(C.POINTER(C.c_int64)), B, T,
                feats.data_ptr(), mask.data_ptr(), None if stats is None else stats.data_ptr(), self._stream()))
        return feats, mask

    def dither_sample(self, B, T):
        """The dither's N(0, 1) draws of utterance rows 0 .. B-1, frames 0 .. T-1: [B, T, W] float32 on the device."""
        torch = _torch()
        W = int(self.options.sample_frequency * 0.001 * self.options.frame_length)
        out = torch.empty((B, T, W), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().lvsr_frontend_dither_sample(self._handle, B, T, out.data_ptr(), self._stream()))
        return out


def _device_stats(cmvn, device, D):
    """The stats of a GlobalCmvn (as they are on the device: no wait) or of a [2, D+1] array, on `device`."""
    torch = _torch()
    if isinstance(cmvn, GlobalCmvn):
        if not cmvn.filled:
            raise ValueError("cmvn stats: no frames yet (accumulate, or set stats with a frame count >= 1)")
        s = cmvn.device_stats
    else:
        s = np.asarray(cmvn, np.float64)
        if s.shape == (2, D + 1) and s[0, D] < 1:
            raise ValueError("cmvn stats: the frame count is %g" % s[0, D])
        s = torch.from_numpy(s)
    if tuple(s.shape) != (2, D + 1):
        raise ValueError("cmvn stats: [2, %d] expected, got %s" % (D + 1, tuple(s.shape)))
    return s.to(device=device, dtype=torch.float64).contiguous()


class GlobalCmvn(object):
    """Kaldi's global CMVN stats [2, D+1] float64 (row 0: column sums | frame count; row 1: sums of squares), kept on
    the front end's device: accumulated over any number of batches, applied with norm_vars.  As Kaldi refuses a
    frame count below 1, they are refused until `accumulate` has run or `stats` has been set with a count >= 1
    (`filled`)."""

    def __init__(self, fbank, stats=None):
        torch = _torch()
        self.fbank = fbank
        D = fbank.feature_dim
        self.device_stats = torch.zeros((2, D + 1), dtype=torch.float64, device=fbank.device)
        self.filled = False
        if stats is not None:
            self.stats = stats

    @property
    def stats(self):
        return self.device_stats.cpu().numpy()

    @stats.setter
    def stats(self, value):
        value = np.asarray(value, np.float64)
        if value.shape != tuple(self.device_stats.shape):
            raise ValueError("cmvn stats: %s expected, got %s" % (tuple(self.device_stats.shape), value.shape))
        self.device_stats.copy_(_torch().from_numpy(value))
        self.filled = bool(value[0, -1] >= 1)

    def save(self, path):
        np.save(path, self.stats)

    @classmethod
    def load(cls, fbank, path):
        return cls(fbank, np.load(path))

    def _args(self, features, mask):
        torch = _torch()
        if not (isinstance(features, torch.Tensor) and features.is_cuda and features.dtype == torch.float32 and
                features.is_contiguous() and features.ndim == 3 and features.shape[2] == self.fbank.feature_dim):
            raise ValueError("features: a contiguous float32 CUDA tensor [T, B, %d] expected" % self.fbank.feature_dim)
        T, B = features.shape[:2]
        if mask is not None:
            mask = mask.to(device=features.device, dtype=torch.float32).contiguous()
            if tuple(mask.shape) != (T, B):
                raise ValueError("mask: [%d, %d] expected" % (T, B))
        return T, B, mask

    def accumulate(self, features, mask=None):
        """Adds the frames of features [T, B, D] whose mask is 1 (None: every frame)."""
        T, B, mask = self._args(features, mask)
        f = self.fbank
        with _torch().cuda.device(f.device):
            _lib.check(_lib.load().lvsr_frontend_accumulate_cmvn(
                f._handle, features.data_ptr(), None if mask is None else mask.data_ptr(), T, B,
                self.device_stats.data_ptr(), f._stream()))
        self.filled = True

    def apply(self, features, mask=None):
        """Normalises features [T, B, D] in place on the frames whose mask is 1; returns them."""
        T, B, mask = self._args(features, mask)
        f = self.fbank
        stats = _device_stats(self, f.device, f.feature_dim)
        with _torch().cuda.device(f.device):
            _lib.check(_lib.load().lvsr_frontend_apply_cmvn(
                f._handle, features.data_ptr(), None if mask is None else mask.data_ptr(), T, B, stats.data_ptr(),
                f._stream()))
        return features
