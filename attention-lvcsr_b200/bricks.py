"""Configuration tokens and initialisation schemes with the reference's names.

The reference's YAML configs instantiate Blocks objects (``!!python/object/apply:
blocks.bricks.Maxout [2]``, ``blocks.initialization.IsotropicGaussian [0.01]`` ...,
lvsr/configs/prototype_speech.yaml, exp/wsj/configs/wsj_jan_new.yaml:25-34).  Here
they are plain value objects: they select a kernel variant or drive the host-side
parameter initialisation; no graph is built.
"""
import numpy as np


class Activation(object):
    kind = "identity"
    num_pieces = 1

    def __repr__(self):
        return "%s()" % type(self).__name__


class Identity(Activation):
    kind = "identity"


class Tanh(Activation):
    kind = "tanh"


class Rectifier(Activation):
    kind = "relu"


class Maxout(Activation):
    """blocks.bricks.Maxout: max over ADJACENT groups of num_pieces features
    (libs/blocks/blocks/bricks/simple.py:160-181)."""
    kind = "maxout"

    def __init__(self, num_pieces=2):
        self.num_pieces = int(num_pieces)

    def __repr__(self):
        return "Maxout(%d)" % self.num_pieces


class GatedRecurrent(object):
    """Transition token: the only transition the CUDA path implements
    (libs/blocks/blocks/bricks/recurrent.py:486-624)."""

    def __init__(self, dim=None, activation=None, gate_activation=None, name=None, **kwargs):
        self.dim = dim
        self.name = name


# ---- initialisation schemes (libs/blocks/blocks/initialization.py:57-208) ------------

class NdarrayInitialization(object):
    def generate(self, rng, shape):
        raise NotImplementedError


class Constant(NdarrayInitialization):
    def __init__(self, constant):
        self.constant = np.asarray(constant)

    def generate(self, rng, shape):
        out = np.empty(shape, dtype=np.float32)
        out[...] = self.constant
        return out


class IsotropicGaussian(NdarrayInitialization):
    def __init__(self, std=1, mean=0):
        self.std, self.mean = std, mean

    def generate(self, rng, shape):
        return rng.normal(self.mean, self.std, size=shape).astype(np.float32)


class Uniform(NdarrayInitialization):
    def __init__(self, mean=0.0, width=None, std=None):
        if (width is not None) == (std is not None):
            raise ValueError("must specify width or std, but not both")
        self.width = np.sqrt(12) * std if std is not None else width
        self.mean = mean

    def __setstate__(self, state):
        # a YAML mapping (`!!python/object:blocks.initialization.Uniform {width: 0.1}`, exp/wsj/configs/
        # wsj_jan_bhd04.yaml) builds the object without __init__: the mapping is taken as the constructor's arguments
        self.__init__(**state)

    def generate(self, rng, shape):
        w = self.width / 2
        return rng.uniform(self.mean - w, self.mean + w, size=shape).astype(np.float32)


class Orthogonal(NdarrayInitialization):
    def __init__(self, scale=1):
        self.scale = scale

    def generate(self, rng, shape):
        if len(shape) != 2:
            raise ValueError("Orthogonal needs a matrix")
        rows, cols = shape
        if rows == cols:
            q, r = np.linalg.qr(rng.randn(rows, cols))
            return (q * np.sign(np.diag(r)) * self.scale).astype(np.float32)
        q1, r1 = np.linalg.qr(rng.randn(rows, rows))
        q2, r2 = np.linalg.qr(rng.randn(cols, cols))
        q1 = q1 * np.sign(np.diag(r1))
        q2 = q2 * np.sign(np.diag(r2))
        k = min(rows, cols)
        return (np.dot(q1[:, :k], q2[:k, :]) * self.scale).astype(np.float32)
