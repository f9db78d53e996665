"""CPU oracle for the attention-lvcsr hot path -- TEST INFRASTRUCTURE ONLY.

This is a NumPy restatement (float64 by default, float32 "twin" on request) of
what the reference's Theano/Blocks graph computes for the path

    pyramidal BiGRU encoder -> content+location attention scan -> GRU decoder
    -> (teacher-forced cost | one generate step | beam search)

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline /
``--impl reference`` legs may import it.  The product path
(``attention-lvcsr_b200``) never does.

Pinning: the reference itself cannot be executed in the build container (Python-2
+ Theano 0.8, see SURVEY.md section 8c), so the oracle is pinned by the
reference's own known-answer tests, restated in ``tests/test_oracle_kat.py``:
conv1d vectors (tests/test_conv1d.py:6-13), GRU step/sequence
(libs/blocks/tests/bricks/test_recurrent.py:432-495), attention freeze sums
113.429 / 415.901 (libs/blocks/tests/bricks/test_attention.py:132-135), sequence
generator freeze sums 482.827 / 16.0942 / 13.5042 / 23.4172 / 199.2402 / -11.6008
(libs/blocks/tests/bricks/test_sequence_generators.py:133-139,254-275) and
``_smallest`` (libs/blocks/tests/test_search.py:65-69).  The location-attention
term, the windowing priors, encoder subsampling and the modified BeamSearch
options are NOT covered by any reference test: for those, parity is
"unpinned by reference tests; pinned by this restated oracle".

Every function cites the reference file:line it follows.  Path prefixes:
  B/  = libs/blocks/blocks/        lvsr/ = lvsr/
All tensors are time-major, exactly as in the reference
(lvsr/datasets/__init__.py:22-29,308).
"""
from __future__ import annotations

import math
from collections import OrderedDict

import numpy as np

# --------------------------------------------------------------------------
# elementary pieces
# --------------------------------------------------------------------------


def sigmoid(x):
    """Logistic; B/bricks/simple.py Logistic -> tensor.nnet.sigmoid."""
    return 1.0 / (1.0 + np.exp(-x))


def log_softmax(x):
    """B/bricks/simple.py:335-337: shifted - log(sum(exp(shifted))) on the last axis."""
    shifted = x - x.max(axis=-1, keepdims=True)
    return shifted - np.log(np.exp(shifted).sum(axis=-1, keepdims=True))


def maxout(x, num_pieces):
    """B/bricks/simple.py:175-181: reshape [..., dim/p, p] and max over the last
    axis, i.e. ADJACENT groups of ``num_pieces`` features."""
    new_shape = x.shape[:-1] + (x.shape[-1] // num_pieces, num_pieces)
    return x.reshape(new_shape).max(axis=-1)


def conv1d(sequences, filters, border_mode="valid"):
    """lvsr/expressions.py:28-54 on top of Theano conv2d (filter_flip=True, i.e.
    a TRUE convolution: libs/Theano/theano/tensor/nnet/opt.py:76-80).

    sequences [B, L], filters [K, w]  ->  [B, K, positions].
    full:  out[b,k,p] = sum_j seq[b, p-j] * filt[k, j],  p in [0, L+w-2]
    valid: the slice of ``full`` where the filter fully overlaps.
    """
    sequences = np.asarray(sequences)
    filters = np.asarray(filters)
    dtype = np.result_type(sequences.dtype, filters.dtype, np.float32)
    B, L = sequences.shape
    K, w = filters.shape
    full = np.zeros((B, K, L + w - 1), dtype=dtype)
    for j in range(w):
        # contribution of filter tap j lands at positions j .. j+L-1
        full[:, :, j:j + L] += sequences[:, None, :] * filters[None, :, j, None]
    if border_mode == "full":
        return full
    if border_mode == "valid":
        return full[:, :, w - 1:L]
    raise ValueError(border_mode)


# --------------------------------------------------------------------------
# recurrent transitions
# --------------------------------------------------------------------------


def gru_step(h, inputs, gate_inputs, state_to_state, state_to_gates, mask=None,
             activation=np.tanh, gate_activation=sigmoid):
    """One GatedRecurrent step, B/bricks/recurrent.py:608-620.

    NOT the cuDNN GRU: the reset gate multiplies the state BEFORE the recurrent
    matmul, gate columns are [update | reset], and h' = c*z + h*(1-z).
    """
    dim = h.shape[-1]
    gate_values = gate_activation(h.dot(state_to_gates) + gate_inputs)
    update_values = gate_values[:, :dim]
    reset_values = gate_values[:, dim:]
    states_reset = h * reset_values
    next_states = activation(states_reset.dot(state_to_state) + inputs)
    next_states = next_states * update_values + h * (1 - update_values)
    if mask is not None:
        next_states = mask[:, None] * next_states + (1 - mask[:, None]) * h
    return next_states


def simple_recurrent_step(h, inputs, W, mask=None, activation=np.tanh):
    """SimpleRecurrent step, B/bricks/recurrent.py:314-328 (used by the KATs only)."""
    next_states = activation(inputs + h.dot(W))
    if mask is not None:
        next_states = mask[:, None] * next_states + (1 - mask[:, None]) * h
    return next_states


def gru_scan(inputs, gate_inputs, mask, p, reverse=False, initial_state=None,
             activation=np.tanh, gate_activation=sigmoid):
    """@recurrent wrapper semantics, B/bricks/recurrent.py:224-231 (theano.scan,
    go_backwards=reverse) + initial state broadcast (:622-624).

    inputs [T,B,D], gate_inputs [T,B,2D], mask [T,B] or None.
    Returns states [T,B,D] in scan order, i.e. for reverse=True states[0] is the
    state after consuming inputs[T-1] (Bidirectional re-reverses, :655-663).
    """
    T, B, D = inputs.shape
    h = (np.repeat(p["initial_state"][None, :], B, 0)
         if initial_state is None else initial_state).astype(inputs.dtype)
    out = np.empty((T, B, D), dtype=inputs.dtype)
    order = range(T - 1, -1, -1) if reverse else range(T)
    for i, t in enumerate(order):
        h = gru_step(h, inputs[t], gate_inputs[t], p["state_to_state"],
                     p["state_to_gates"], None if mask is None else mask[t],
                     activation, gate_activation)
        out[i] = h
    return out


def linear(x, W, b=None):
    """B/bricks/simple.py:73-76."""
    # 2-D BLAS product (numpy's N-D dot falls off the gemm path)
    y = np.ascontiguousarray(x).reshape(-1, x.shape[-1]).dot(W).reshape(x.shape[:-1] + (W.shape[1],))
    if b is not None:
        y = y + b
    return y


# --------------------------------------------------------------------------
# parameter naming (Blocks brick paths) -- SURVEY.md section 8b
# --------------------------------------------------------------------------

DEFAULT_PRIOR = dict(type="expanding", initial_begin=0, initial_end=10000,
                     min_speed=0, max_speed=0)  # lvsr/bricks/attention.py:72-74


def make_config(num_features=40, dims_bidir=(256, 256, 256, 256), subsample=None,
                dim_dec=256, dim_matcher=None, conv_n=100, conv_num_filters=10,
                num_phonemes=32, post_merge_dims=None, maxout_pieces=2,
                dim_output_embedding=None, prior=None, energy_normalizer="softmax",
                attention_type="content_and_conv", eos_label=None,
                max_decoded_length_scale=1.0, use_states_for_readout=True,
                post_merge_activation=None, embed_outputs=True):
    """The subset of ``config['net']`` the hot path depends on
    (lvsr/bricks/recognizer.py:176-204)."""
    dims_bidir = list(dims_bidir)
    cfg = dict(
        num_features=int(num_features),
        dims_bidir=dims_bidir,
        subsample=list(subsample) if subsample else [1] * len(dims_bidir),
        dim_dec=int(dim_dec),
        dim_matcher=int(dim_matcher if dim_matcher is not None else dim_dec),  # :225-226
        conv_n=int(conv_n), conv_num_filters=int(conv_num_filters),
        num_phonemes=int(num_phonemes),
        post_merge_dims=list(post_merge_dims) if post_merge_dims else [int(dim_dec)],
        maxout_pieces=int(maxout_pieces) if (post_merge_activation in (None, "maxout")) else 1,
        post_merge_activation=(post_merge_activation or ("maxout" if maxout_pieces > 1 else "relu")),
        # LookupFeedback(V+1, dim) | OneOfNFeedback(V+1): the feedback is the one-hot vector (recognizer.py:278-284)
        dim_feedback=(int(dim_output_embedding if dim_output_embedding is not None else dim_dec) if embed_outputs
                      else int(num_phonemes) + 1),
        embed_outputs=bool(embed_outputs),
        prior=dict(prior) if prior else dict(DEFAULT_PRIOR),
        energy_normalizer=energy_normalizer or "softmax",
        attention_type=attention_type,
        eos_label=int(eos_label if eos_label is not None else num_phonemes - 1),
        max_decoded_length_scale=float(max_decoded_length_scale),
        use_states_for_readout=bool(use_states_for_readout),
    )
    assert cfg["attention_type"] == "content_and_conv"
    assert len(cfg["post_merge_dims"]) == 1
    return cfg


def dim_encoded(cfg):
    return 2 * cfg["dims_bidir"][-1]


def param_shapes(cfg):
    """Parameter names + shapes in Blocks initialisation order (children depth
    first, then own ``_initialize``: B/bricks/base.py:642-666; recognizer children
    = [encoder, top, bottom, generator]: lvsr/bricks/recognizer.py:349).
    Names are Blocks parameter paths (B/select.py:160-220)."""
    shapes = OrderedDict()
    din = cfg["num_features"]
    for l, D in enumerate(cfg["dims_bidir"]):
        for d in ("forward", "backward"):
            base = "/recognizer/encoder/bidir%d/%s" % (l, d)
            # RecurrentWithFork.children = [recurrent.brick, fork] (lvsr/bricks/__init__.py:31)
            shapes[base + "/gatedrecurrent.state_to_state"] = (D, D)
            shapes[base + "/gatedrecurrent.state_to_gates"] = (D, 2 * D)
            shapes[base + "/gatedrecurrent.initial_state"] = (D,)
            shapes[base + "/fork/fork_inputs.b"] = (D,)
            shapes[base + "/fork/fork_inputs.W"] = (din, D)
            shapes[base + "/fork/fork_gate_inputs.b"] = (2 * D,)
            shapes[base + "/fork/fork_gate_inputs.W"] = (din, 2 * D)
        din = 2 * D
    E, C, M = dim_encoded(cfg), cfg["dim_dec"], cfg["dim_matcher"]
    K, w = cfg["conv_num_filters"], 2 * cfg["conv_n"] + 1
    V, Cfb, Cpm = cfg["num_phonemes"], cfg["dim_feedback"], cfg["post_merge_dims"][0]
    g = "/recognizer/generator"
    # generator.children = [readout, fork, transition] (B/bricks/sequence_generators.py:157)
    if cfg.get("embed_outputs", True):
        shapes[g + "/readout/lookupfeedback/lookuptable.W"] = (V + 1, Cfb)
    if cfg["use_states_for_readout"]:
        shapes[g + "/readout/merge/transform_states.W"] = (C, Cpm)
    shapes[g + "/readout/merge/transform_weighted_averages.W"] = (E, Cpm)
    shapes[g + "/readout/post_merge/bias.b"] = (Cpm,)
    shapes[g + "/readout/post_merge/mlp/linear_0.b"] = (V,)
    shapes[g + "/readout/post_merge/mlp/linear_0.W"] = (Cpm // cfg["maxout_pieces"], V)
    shapes[g + "/fork/fork_inputs.b"] = (C,)
    shapes[g + "/fork/fork_inputs.W"] = (Cfb, C)
    shapes[g + "/fork/fork_gate_inputs.b"] = (2 * C,)
    shapes[g + "/fork/fork_gate_inputs.W"] = (Cfb, 2 * C)
    a = g + "/att_trans"
    shapes[a + "/transition.state_to_state"] = (C, C)
    shapes[a + "/transition.state_to_gates"] = (C, 2 * C)
    shapes[a + "/transition.initial_state"] = (C,)
    shapes[a + "/conv_att/state_trans/transform_states.W"] = (C, M)
    shapes[a + "/conv_att/preprocess.b"] = (M,)
    shapes[a + "/conv_att/preprocess.W"] = (E, M)
    if cfg["energy_normalizer"] != "softmax":
        shapes[a + "/conv_att/energy_comp/linear.b"] = (1,)  # lvsr/bricks/attention.py:67-70
    shapes[a + "/conv_att/energy_comp/linear.W"] = (M, 1)
    shapes[a + "/conv_att/handler.W"] = (K, M)
    shapes[a + "/conv_att/conv1d.filters"] = (K, w)
    shapes[a + "/distribute/fork_inputs.W"] = (E, C)
    shapes[a + "/distribute/fork_gate_inputs.W"] = (E, 2 * C)
    return shapes


def orthogonal(rng, shape, scale=1.0):
    """B/initialization.py:185-208 (square case :190-195)."""
    if shape[0] == shape[1]:
        M = rng.randn(*shape)
        Q, R = np.linalg.qr(M)
        Q = Q * np.sign(np.diag(R))
        return Q * scale
    M1 = rng.randn(shape[0], shape[0])
    M2 = rng.randn(shape[1], shape[1])
    Q1, R1 = np.linalg.qr(M1)
    Q2, R2 = np.linalg.qr(M2)
    Q1 = Q1 * np.sign(np.diag(R1))
    Q2 = Q2 * np.sign(np.diag(R2))
    n_min = min(shape)
    return np.dot(Q1[:, :n_min], Q2[:n_min, :]) * scale


def init_params(cfg, seed=1, weights_std=0.01, initial_state_std=0.001,
                scale=1.0, dtype=np.float64):
    """WSJ initialisation scheme (exp/wsj/configs/wsj_jan_new.yaml:25-34):
    IsotropicGaussian(weights_std) weights, zero biases, Orthogonal recurrent
    weights (state_to_state AND both gate blocks: lvsr/bricks/recognizer.py:363-373
    pushes rec_weights_init as weights_init onto every BaseRecurrent),
    IsotropicGaussian(initial_state_std) initial states; one shared
    RandomState(seed) in brick order (B/bricks/interfaces.py:157-162).
    ``scale`` multiplies every non-recurrent weight: the "trained-like" parameter
    set of SURVEY.md section 8d uses scale=10.
    """
    rng = np.random.RandomState(seed)
    out = OrderedDict()
    for name, shape in param_shapes(cfg).items():
        leaf = name.rsplit(".", 1)[1]
        if leaf == "b":
            v = np.zeros(shape)
        elif leaf == "state_to_state":
            v = orthogonal(rng, shape)
        elif leaf == "state_to_gates":
            D = shape[0]
            v = np.hstack([orthogonal(rng, (D, D)), orthogonal(rng, (D, D))])  # recurrent.py:576-579
        elif leaf == "initial_state":
            v = rng.normal(0, initial_state_std, size=shape) * scale
        else:
            v = rng.normal(0, weights_std, size=shape) * scale
        out[name] = np.ascontiguousarray(v, dtype=dtype)
    return out


def cast_params(params, dtype):
    return OrderedDict((k, np.ascontiguousarray(v, dtype=dtype)) for k, v in params.items())


# --------------------------------------------------------------------------
# encoder
# --------------------------------------------------------------------------


def _gru_params(params, base):
    return dict(state_to_state=params[base + ".state_to_state"],
                state_to_gates=params[base + ".state_to_gates"],
                initial_state=params[base + ".initial_state"])


def recurrent_with_fork(x, mask, params, base, reverse, activation=np.tanh, gate_activation=sigmoid):
    """lvsr/bricks/__init__.py:39-43: Fork(Linear) over the WHOLE sequence, then the scan.
    (The activations are arguments only so the reference's Tanh-gated known-answer test can be
    driven through this very function; the recognizer always uses tanh / logistic.)"""
    a = linear(x, params[base + "/fork/fork_inputs.W"], params[base + "/fork/fork_inputs.b"])
    g = linear(x, params[base + "/fork/fork_gate_inputs.W"], params[base + "/fork/fork_gate_inputs.b"])
    return gru_scan(a, g, mask, _gru_params(params, base + "/gatedrecurrent"), reverse=reverse,
                    activation=activation, gate_activation=gate_activation)


def bidirectional(x, mask, params, base, **act):
    """B/bricks/recurrent.py:655-663: forward scan; backward scan with
    reverse=True then [::-1]; concatenate on the feature axis, forward first."""
    fwd = recurrent_with_fork(x, mask, params, base + "/forward", reverse=False, **act)
    bwd = recurrent_with_fork(x, mask, params, base + "/backward", reverse=True, **act)[::-1]
    return np.concatenate([fwd, bwd], axis=2)


def encoder(cfg, params, x, mask=None, return_layers=False, **act):
    """lvsr/bricks/__init__.py:71-78.  x [T,B,F], mask [T,B] -> (encoded [T',B,E],
    encoded_mask [T',B]).  Subsampling x[::k] happens AFTER the full-rate layer."""
    layers = []
    for l, k in enumerate(cfg["subsample"]):
        x = bidirectional(x, mask, params, "/recognizer/encoder/bidir%d" % l, **act)
        x = x[::k]
        if mask is not None:
            mask = mask[::k]
        layers.append(x)
    enc_mask = mask if mask is not None else np.ones_like(x[:, :, 0])
    if return_layers:
        return x, enc_mask, layers
    return x, enc_mask


# --------------------------------------------------------------------------
# attention
# --------------------------------------------------------------------------

_ATT = "/recognizer/generator/att_trans/conv_att"


def preprocess(params, attended):
    """lvsr/bricks/attention.py:228-230."""
    return linear(attended, params[_ATT + "/preprocess.W"], params[_ATT + "/preprocess.b"])


def compute_weights(energies, mask, normalizer="softmax"):
    """lvsr/bricks/attention.py:191-213.  energies/mask [Tw,B].  The max runs over
    ALL window positions (masked ones too) and the normaliser gains +1 where a
    column's mask is all zero."""
    if normalizer == "softmax":
        energies = energies - energies.max(axis=0)
        unnorm = np.exp(energies)
    elif normalizer == "logistic":
        unnorm = sigmoid(energies)
    elif normalizer == "relu":
        unnorm = np.maximum(energies / 1000.0, 0.0)
    else:
        raise ValueError(normalizer)
    unnorm = unnorm * mask
    normalization = unnorm.sum(axis=0) + np.all(1 - mask, axis=0)
    return unnorm / normalization



def content_take_glimpses(attended, preprocessed, attended_mask, states, W_state, v):
    """SequenceContentAttention.take_glimpses (content-only attention),
    B/bricks/attention.py:331-388 -- used by the reference KATs that pin
    compute_weights / weighted averages / AttentionRecurrent step order."""
    match = preprocessed + states.dot(W_state)[None]
    e = np.tanh(match).dot(v)[..., 0]
    w = compute_weights(e, attended_mask, "softmax")
    return (w[:, :, None] * attended).sum(axis=0), w.T


def compute_energies(cfg, params, P_cut, weights_cut, states):
    """lvsr/bricks/attention.py:98-114.  P_cut [Tw,B,M], weights_cut [B,Tw], states [B,C]."""
    n = cfg["conv_n"]
    match = P_cut + states.dot(params[_ATT + "/state_trans/transform_states.W"])[None]
    conv_result = conv1d(weights_cut, params[_ATT + "/conv1d.filters"], "full")   # [B,K,Tw+2n]
    feats = conv_result[:, :, n:conv_result.shape[2] - n].transpose(0, 2, 1)      # [B,Tw,K]
    match = match + feats.dot(params[_ATT + "/handler.W"]).transpose(1, 0, 2)
    e = np.tanh(match).dot(params[_ATT + "/energy_comp/linear.W"])[..., 0]
    if cfg["energy_normalizer"] != "softmax":
        e = e + params[_ATT + "/energy_comp/linear.b"][0]
    return e


def attention_window(cfg, length, weights, step):
    """Window selection of take_glimpses, lvsr/bricks/attention.py:123-163.
    Returns (begin, end, additional_mask [B,Tw] or None)."""
    p = cfg["prior"]
    ptype = p.get("type", "expanding")
    if ptype == "expanding":
        begin = p["initial_begin"] + step[0] * p["min_speed"]
        end = p["initial_end"] + step[0] * p["max_speed"]
        begin = max(0, min(length - 1, begin))
        end = max(0, min(length, end))
        add_mask = None
    elif ptype.startswith("window_around"):
        if ptype == "window_around_mean":
            pos = (weights * np.arange(length, dtype=weights.dtype)[None, :]).sum(axis=1)
        elif ptype == "window_around_median":
            ali = ((np.cumsum(weights, axis=1) - 0.5) >= 0).astype(np.int8)
            pos = np.argmax(ali[:, 1:] - ali[:, :-1], axis=1)
        else:
            raise ValueError(ptype)
        begins = np.floor(pos - p["before"])
        ends = np.ceil(pos + p["after"])
        begin = int(max(0, begins.min()))
        end = int(min(length, ends.max()))
        position_cut = np.arange(begin * 1.0, end * 1.0, 1.0, dtype=weights.dtype)[None, :]
        add_mask = ((position_cut > begins[:, None]) *
                    (position_cut < ends[:, None])).astype(weights.dtype)
    else:
        raise Exception("Unknown prior type: %s" % ptype)
    begin = int(math.floor(begin))
    end = int(math.ceil(end))
    return begin, end, add_mask


def take_glimpses(cfg, params, attended, preprocessed, attended_mask, weights, step, states):
    """SequenceContentAndConvAttention.take_glimpses, lvsr/bricks/attention.py:120-183.
    attended [T',B,E], preprocessed [T',B,M] (or None -> recomputed, :101-102),
    attended_mask [T',B], weights [B,T'], step [B] int64, states [B,C].
    -> weighted_averages [B,E], weights [B,T'], energies [B,T'], step+1."""
    length = attended.shape[0]
    begin, end, add_mask = attention_window(cfg, length, weights, step)
    if preprocessed is None:
        preprocessed = preprocess(params, attended)
    att_cut = attended[begin:end]
    P_cut = preprocessed[begin:end]
    mask_cut = attended_mask[begin:end] * (add_mask.T if add_mask is not None else 1)
    weights_cut = weights[:, begin:end]
    e_cut = compute_energies(cfg, params, P_cut, weights_cut, states)
    w_cut = compute_weights(e_cut, mask_cut, cfg["energy_normalizer"])
    weighted_averages = (w_cut[:, :, None] * att_cut).sum(axis=0)      # B/bricks/attention.py:256
    new_weights = np.zeros_like(weights.T)
    new_energies = np.zeros_like(weights.T)
    new_weights[begin:end] = w_cut
    new_energies[begin:end] = e_cut
    return weighted_averages, new_weights.T, new_energies.T, step + 1


def initial_glimpses(cfg, batch_size, attended):
    """lvsr/bricks/attention.py:215-222: zeros, one-hot(0) weights AND energies, step 0."""
    Tl = attended.shape[0]
    onehot = np.zeros((batch_size, Tl), dtype=attended.dtype)
    onehot[:, 0] = 1
    return (np.zeros((batch_size, dim_encoded(cfg)), dtype=attended.dtype),
            onehot.copy(), onehot.copy(), np.zeros((batch_size,), dtype=np.int64))


# --------------------------------------------------------------------------
# decoder: transition, readout, cost, generate step
# --------------------------------------------------------------------------

_GEN = "/recognizer/generator"
_TR = _GEN + "/att_trans"


def compute_states(cfg, params, states, inputs, gate_inputs, weighted_averages, mask=None):
    """AttentionRecurrent.compute_states, B/bricks/attention.py:625-662: Distribute
    adds ctx.W (no bias) to both sequence inputs (B/bricks/parallel.py:249-265),
    then the wrapped GRU step."""
    inputs = weighted_averages.dot(params[_TR + "/distribute/fork_inputs.W"]) + inputs
    gate_inputs = weighted_averages.dot(params[_TR + "/distribute/fork_gate_inputs.W"]) + gate_inputs
    return gru_step(states, inputs, gate_inputs,
                    params[_TR + "/transition.state_to_state"],
                    params[_TR + "/transition.state_to_gates"], mask)


def feedback_fork(cfg, params, outputs):
    """readout.feedback (LookupFeedback, B/bricks/sequence_generators.py:839-842)
    followed by generator.fork (Linear+bias each)."""
    if cfg.get("embed_outputs", True):
        fb = params[_GEN + "/readout/lookupfeedback/lookuptable.W"][outputs]
    else:       # OneOfNFeedback.feedback, lvsr/bricks/__init__.py:97-104: eye(V+1)[outputs]
        fb = np.eye(cfg["num_phonemes"] + 1, dtype=params[_GEN + "/fork/fork_inputs.W"].dtype)[outputs]
    inputs = linear(fb, params[_GEN + "/fork/fork_inputs.W"], params[_GEN + "/fork/fork_inputs.b"])
    gate_inputs = linear(fb, params[_GEN + "/fork/fork_gate_inputs.W"],
                         params[_GEN + "/fork/fork_gate_inputs.b"])
    return inputs, gate_inputs


def readout(cfg, params, states, weighted_averages):
    """Readout.readout, B/bricks/sequence_generators.py:614-619 with the post_merge
    of lvsr/bricks/recognizer.py:298-320: Merge (no biases) -> Bias -> Maxout(2)
    (or ReLU) -> Linear."""
    r = weighted_averages.dot(params[_GEN + "/readout/merge/transform_weighted_averages.W"])
    if cfg["use_states_for_readout"]:
        r = r + states.dot(params[_GEN + "/readout/merge/transform_states.W"])
    r = r + params[_GEN + "/readout/post_merge/bias.b"]
    act = cfg["post_merge_activation"]
    if act == "maxout":
        r = maxout(r, cfg["maxout_pieces"])
    elif act == "relu":
        r = np.maximum(r, 0)
    elif act == "tanh":            # the reference default, lvsr/bricks/recognizer.py:206-207
        r = np.tanh(r)
    elif act != "identity":
        raise ValueError(act)
    return linear(r, params[_GEN + "/readout/post_merge/mlp/linear_0.W"],
                  params[_GEN + "/readout/post_merge/mlp/linear_0.b"])


def initial_states(cfg, params, batch_size, attended):
    """BaseSequenceGenerator.initial_states, B/bricks/sequence_generators.py:408-421;
    y_0 = num_phonemes (lvsr/bricks/recognizer.py:286)."""
    s0 = np.repeat(params[_TR + "/transition.initial_state"][None, :], batch_size, 0).astype(attended.dtype)
    wa, w, e, step = initial_glimpses(cfg, batch_size, attended)
    return OrderedDict(states=s0,
                       outputs=np.full((batch_size,), cfg["num_phonemes"], dtype=np.int64),
                       weighted_averages=wa, weights=w, energies=e, step=step)


def cost_matrix(cfg, params, attended, attended_mask, labels, labels_mask=None,
                return_all=False):
    """BaseSequenceGenerator.evaluate / cost_matrix, B/bricks/sequence_generators.py:254-326.
    labels [L,B] int64, labels_mask [L,B] or None.  Teacher forcing: glimpses come
    from the PREVIOUS state; readout sees s_{i-1} and ctx_i (:294-299).  The label
    mask freezes only the GRU state (quirk 11)."""
    L, B = labels.shape
    P = preprocess(params, attended)                         # hoisted once: B/bricks/attention.py:733-738
    inputs, gate_inputs = feedback_fork(cfg, params, labels)  # [L,B,C], [L,B,2C]
    st = initial_states(cfg, params, B, attended)
    s, wa, w, e, step = st["states"], st["weighted_averages"], st["weights"], st["energies"], st["step"]
    states_prev, glimpses = [], []
    all_w, all_e = [], []
    for i in range(L):
        states_prev.append(s)
        wa, w, e, step = take_glimpses(cfg, params, attended, P, attended_mask, w, step, s)
        s = compute_states(cfg, params, s, inputs[i], gate_inputs[i], wa,
                           None if labels_mask is None else labels_mask[i])
        glimpses.append(wa)
        all_w.append(w)
        all_e.append(e)
    states_prev = np.stack(states_prev)        # results['states'][:-1]
    ctx = np.stack(glimpses)                   # results['weighted_averages'][1:]
    readouts = readout(cfg, params, states_prev, ctx)
    logp = log_softmax(readouts)
    costs = -np.take_along_axis(logp, labels[..., None], axis=-1)[..., 0]   # simple.py:361-364
    if labels_mask is not None:
        costs = costs * labels_mask
    if return_all:
        return dict(costs=costs, states=states_prev, weighted_averages=ctx,
                    weights=np.stack(all_w), energies=np.stack(all_e), final_state=s)
    return costs


def recognizer_cost(cfg, params, recordings, recordings_mask, labels, labels_mask, return_all=False):
    """SpeechRecognizer.cost, lvsr/bricks/recognizer.py:375-390 (bottom/top = Identity)."""
    attended, attended_mask = encoder(cfg, params, recordings, recordings_mask)
    return cost_matrix(cfg, params, attended, attended_mask, labels, labels_mask, return_all)


def batch_cost(costs):
    """lvsr/main.py:340-345: sum over time and batch, divided by the batch size."""
    return costs.sum() / costs.shape[1]


def analyze(cfg, params, recordings, groundtruth, prediction=None):
    """SpeechRecognizer.analyze, lvsr/bricks/recognizer.py:452-494: batch of one,
    mask of ones (single_to_batch_inputs :145-151), no label mask.
    -> costs [L], weights [L,T'], energies [L,T']."""
    x = recordings[:, None, :]
    m = np.ones(x.shape[:2], dtype=x.dtype)
    labels = (groundtruth if prediction is None else prediction)[:, None]
    r = recognizer_cost(cfg, params, x, m, labels, None, return_all=True)
    return r["costs"][:, 0], r["weights"][:, 0, :], r["energies"][:, 0, :]


# ---- the four BeamSearch functions (B/search.py:97-142) ---------------------


def context_computer(cfg, params, recordings):
    """recordings [T,B,F] -> (attended, attended_mask); search uses use_mask=False
    (lvsr/bricks/recognizer.py:503) so the encoder runs unmasked and the mask is ones."""
    return encoder(cfg, params, recordings, None)


def logprobs_computer(cfg, params, attended, attended_mask, st):
    """-log p(y | state) for every y: take_glimpses (preprocess recomputed, see
    SURVEY.md 3.2) -> readout(s_{i-1}, ctx_i) -> SoftmaxEmitter.costs
    (B/bricks/sequence_generators.py:346-355,790-792)."""
    wa, _, _, _ = take_glimpses(cfg, params, attended, None, attended_mask,
                                st["weights"], st["step"], st["states"])
    return -log_softmax(readout(cfg, params, st["states"], wa))


def next_state_computer(cfg, params, attended, attended_mask, st, outputs):
    """generate() with the emitted symbols given, B/bricks/sequence_generators.py:346-377."""
    wa, w, e, step = take_glimpses(cfg, params, attended, None, attended_mask,
                                   st["weights"], st["step"], st["states"])
    inputs, gate_inputs = feedback_fork(cfg, params, outputs)
    s = compute_states(cfg, params, st["states"], inputs, gate_inputs, wa, None)
    return OrderedDict(states=s, outputs=np.asarray(outputs, dtype=np.int64),
                       weighted_averages=wa, weights=w, energies=e, step=step)


def generate_greedy(cfg, params, attended, attended_mask, n_steps):
    """generate() iterated with argmax emission (the deterministic stand-in for
    SoftmaxEmitter.emit's multinomial; equals beam_size=1 search without the stop logic)."""
    B = attended.shape[1]
    st = initial_states(cfg, params, B, attended)
    outs, costs = [], []
    for _ in range(n_steps):
        lp = logprobs_computer(cfg, params, attended, attended_mask, st)
        y = lp.argmin(axis=1)
        costs.append(lp[np.arange(B), y])
        st = next_state_computer(cfg, params, attended, attended_mask, st, y)
        outs.append(y)
    return np.stack(outs), np.stack(costs), st


# --------------------------------------------------------------------------
# beam search (B/search.py:220-407), quirks of SURVEY.md section 8a item 7 kept
# --------------------------------------------------------------------------


class CandidateNotFoundError(Exception):
    """B/search.py:15-16."""


def smallest(matrix, k):
    """BeamSearch._smallest, B/search.py:220-242: argpartition, then argsort of the
    k survivors (tie order is numpy's)."""
    flat = matrix.flatten()
    if flat.shape[0] > k:
        args = np.argpartition(flat, k)[:k]
    else:
        args = np.arange(flat.shape[0])
    args = args[np.argsort(flat[args])]
    return np.unravel_index(args, matrix.shape), flat[args]


def _take_states(st, idx):
    return OrderedDict((k, np.take(v, idx, axis=0)) for k, v in st.items())


def beam_search(cfg, params, recordings, beam_size, eol_symbol=None, max_length=None,
                ignore_first_eol=False, char_discount=0, round_to_inf=1e9,
                stop_on="patience", validate_solution_function=None,
                computers=None, as_arrays=False, stats=None):
    """BeamSearch.search for ONE utterance, B/search.py:244-407, driven the way
    SpeechRecognizer.beam_search does (lvsr/bricks/recognizer.py:513-533):
    recordings [T,F] -> batch axis inserted, max_length = int(T / scale).

    ``computers`` lets a test substitute the four device functions (same
    signatures as the oracle's) while keeping this host logic as the checker.
    ``stats`` (a dict) receives what the settings decided: "steps" run, "stop"
    ("patience" / "optimistic" when a criterion ended the loop, else None),
    "finished" (hypotheses added to done), "eol_removed" (eol hypotheses whose
    step cost reached round_to_inf), "eol_kept_first" (eol hypotheses kept in
    the beam at step 0 by ignore_first_eol) and "rejected" (by the validator).

    The ranking key is float64 whatever the cost dtype, as under numpy 1.x
    where the reference ran (a float32 scalar minus a Python float was
    float64 there; NEP 50 makes it float32).
    """
    if stats is not None:
        stats.update(steps=0, stop=None, finished=0, eol_removed=0, eol_kept_first=0, rejected=0)
    c = computers or {}
    f_ctx = c.get("context", lambda x: context_computer(cfg, params, x))
    f_init = c.get("initial", lambda att: initial_states(cfg, params, 1, att))
    f_logp = c.get("logprobs", lambda att, m, st: logprobs_computer(cfg, params, att, m, st))
    f_next = c.get("next", lambda att, m, st, y: next_state_computer(cfg, params, att, m, st, y))
    if eol_symbol is None:
        eol_symbol = cfg["eos_label"]
    if max_length is None:
        max_length = int(recordings.shape[0] / cfg["max_decoded_length_scale"])

    attended, attended_mask = f_ctx(recordings[:, None, :])
    big_att, big_mask = attended, attended_mask
    st = f_init(attended)

    all_outputs = st["outputs"][None, :]
    all_costs = np.zeros(all_outputs.shape, dtype=attended.dtype)
    done = []
    min_cost = 1000
    patience = None

    def rank(item):
        return float(item[1][-1]) - char_discount * len(item[1])

    for i in range(max_length):
        width = st["states"].shape[0]
        if width == 0:
            break
        if stop_on == "patience":
            done = sorted(done, key=rank)[:beam_size]
            if done:
                best = rank(done[0])
                if best < min_cost:
                    min_cost = best
                    patience = 30
                else:
                    patience -= 1
                    if patience == 0:
                        if stats is not None:
                            stats["stop"] = "patience"
                        break
        elif stop_on == "optimistic_future_cost":
            if len(done) >= beam_size:
                optimistic = float(all_costs[-1, :].min()) - char_discount * max_length
                if rank(done[beam_size - 1]) < optimistic:
                    if stats is not None:
                        stats["stop"] = "optimistic"
                    break
        else:
            raise ValueError("Unknown stopping criterion {}".format(stop_on))

        if big_att.shape[1] != width:
            big_att = np.take(attended, [0] * width, axis=1)
            big_mask = np.take(attended_mask, [0] * width, axis=1)
        logprobs = f_logp(big_att, big_mask, st)
        assert np.isfinite(logprobs).all()
        next_costs = all_costs[-1, :, None] + logprobs
        (indexes, outputs), chosen_costs = smallest(next_costs, beam_size)

        st = _take_states(st, indexes)
        all_outputs = np.take(all_outputs, indexes, axis=1)
        all_costs = np.take(all_costs, indexes, axis=1)
        width = st["states"].shape[0]
        if big_att.shape[1] != width:
            big_att = np.take(attended, [0] * width, axis=1)
            big_mask = np.take(attended_mask, [0] * width, axis=1)
        st = f_next(big_att, big_mask, st, outputs)

        all_outputs = np.vstack([all_outputs, outputs[None, :]])
        all_costs = np.vstack([all_costs, chosen_costs[None, :]])

        mask = outputs != eol_symbol
        if ignore_first_eol and i == 0:
            mask[:] = 1
        finished = np.where((all_outputs[-1] == eol_symbol) &
                            (all_costs[-1] - all_costs[-2] < round_to_inf))[0]
        for idx in finished:
            if (validate_solution_function is None or
                    validate_solution_function(recordings, all_outputs[:, idx])):
                done.append((all_outputs[:, idx], all_costs[:, idx]))
                if stats is not None:
                    stats["finished"] += 1
            elif stats is not None:
                stats["rejected"] += 1
        if stats is not None:
            n_eol = int(np.count_nonzero(all_outputs[-1] == eol_symbol))
            stats["steps"] = i + 1
            stats["eol_removed"] += n_eol - len(finished)
            if ignore_first_eol and i == 0:
                stats["eol_kept_first"] += n_eol
        unfinished = np.where(mask == 1)[0]
        st = _take_states(st, unfinished)
        all_outputs = np.take(all_outputs, unfinished, axis=1)
        all_costs = np.take(all_costs, unfinished, axis=1)

    if not done:
        raise CandidateNotFoundError()
    done = sorted(done, key=rank)
    if as_arrays:
        return done
    # result_to_lists (:401-407): strip the initial symbol, total cost = last cumulative cost
    outs = [[int(t) for t in seq[1:]] for seq, _ in done]
    costs = [float(cost[-1]) for _, cost in done]
    return outs, costs


# --------------------------------------------------------------------------
# synthetic workloads (SURVEY.md section 8d)
# --------------------------------------------------------------------------


def synthetic_batch(cfg, B, T, seed=1234, dtype=np.float64, label_div=8, min_frac=0.6):
    """RandomState(seed): lengths U{ceil(0.6T)..T} with max == T, right-padded 0/1
    masks, N(0,1) features, labels U{0..V-2} of length ceil(T_b/8) with eos appended."""
    rng = np.random.RandomState(seed)
    V = cfg["num_phonemes"]
    lens = rng.randint(int(math.ceil(min_frac * T)), T + 1, size=B)
    lens[rng.randint(B)] = T
    x = rng.normal(size=(T, B, cfg["num_features"]))
    m = (np.arange(T)[:, None] < lens[None, :]).astype(dtype)
    x = (x * m[:, :, None]).astype(dtype)
    lab_lens = np.ceil(lens / float(label_div)).astype(int) + 1
    L = int(lab_lens.max())
    labels = np.zeros((L, B), dtype=np.int64)
    lm = np.zeros((L, B), dtype=dtype)
    for b in range(B):
        n = lab_lens[b]
        labels[:n - 1, b] = rng.randint(0, V - 1, size=n - 1)
        labels[n - 1, b] = cfg["eos_label"]
        lm[:n, b] = 1
    return x, m, labels, lm
