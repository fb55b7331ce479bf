"""Parameter table of the 4-point regressor (flat fp32 buffer layout + initialisation).

The network is the reference's `HomographyModel._vgg` (code/homography_model.py:107-133):
8 x (3x3 conv + bias + ReLU), 3 x maxpool 2x2, fc1 32768->1024 + ReLU, fc2 1024->8.
Variable names and shapes are the reference's TF-Slim checkpoint names
(scopes at code/homography_model.py:358,108-131,97-98): conv kernels are HWIO, fully
connected kernels are [in, out]; the flatten order in front of fc1 is NHWC.

Everything lives in ONE flat fp32 buffer (params / grads / Adam m / Adam v share this layout),
so the data-parallel gradient mean is a single allreduce over one contiguous range
(reference: utils/utils.py:380-403 `get_average_grads`) and Adam is a single fused launch.
"""
from collections import OrderedDict, namedtuple

import numpy as np

ParamSpec = namedtuple("ParamSpec", "name shape offset size fan_in fan_out")

# (scope, cin, cout) of the 8 convolutions in forward order; spatial size of the layer input.
CONV_LAYERS = [
    ("model/conv_block1/conv1", 2, 64, 128),
    ("model/conv_block1/conv2", 64, 64, 128),
    ("model/conv_block2/conv1", 64, 64, 64),
    ("model/conv_block2/conv2", 64, 64, 64),
    ("model/conv_block3/conv1", 64, 128, 32),
    ("model/conv_block3/conv2", 128, 128, 32),
    ("model/conv_block4/conv1", 128, 128, 16),
    ("model/conv_block4/conv2", 128, 128, 16),
]
FC_LAYERS = [
    ("model/fc1/fc1", 16 * 16 * 128, 1024),
    ("model/fc2/fc2", 1024, 8),
]


def param_specs(patch_size=128):
    """Ordered table name -> ParamSpec. Offsets are in floats; every tensor starts 128-byte aligned."""
    assert patch_size % 8 == 0
    specs = OrderedDict()
    off = 0

    def add(name, shape, fan_in, fan_out):
        nonlocal off
        size = int(np.prod(shape))
        specs[name] = ParamSpec(name, tuple(shape), off, size, fan_in, fan_out)
        off += (size + 31) // 32 * 32

    for scope, cin, cout, _ in CONV_LAYERS:
        add(scope + "/weights", (3, 3, cin, cout), 9 * cin, 9 * cout)
        add(scope + "/biases", (cout,), 0, 0)
    feat = (patch_size // 8) * (patch_size // 8) * 128
    add("model/fc1/fc1/weights", (feat, 1024), feat, 1024)
    add("model/fc1/fc1/biases", (1024,), 0, 0)
    add("model/fc2/fc2/weights", (1024, 8), 1024, 8)
    add("model/fc2/fc2/biases", (8,), 0, 0)
    return specs


def total_floats(specs):
    last = next(reversed(specs.values()))
    return last.offset + (last.size + 31) // 32 * 32


def num_parameters(specs):
    return sum(s.size for s in specs.values())


def init_flat(seed, patch_size=128):
    """TF-Slim defaults (third-party, not in /root/reference; call sites homography_model.py:91,128,131):
    weights Xavier-uniform  U(-l, l), l = sqrt(6 / (fan_in + fan_out)); biases zero."""
    specs = param_specs(patch_size)
    flat = np.zeros(total_floats(specs), dtype=np.float32)
    rng = np.random.default_rng(seed)
    chunk = 1 << 24          # float64 draws per call: the same stream as one call, without a float64 copy of fc1 (32 GB at P = 1408)
    for s in specs.values():
        if s.fan_in:
            lim = np.sqrt(6.0 / (s.fan_in + s.fan_out))
            for a in range(0, s.size, chunk):
                b = min(s.size, a + chunk)
                flat[s.offset + a:s.offset + b] = rng.uniform(-lim, lim, size=b - a).astype(np.float32)
    return flat


def init_flat_large(seed, patch_size=128, fc2_gain=600.0, bias_amp=0.05, out_bias=20.0):
    """Seeded "large-output" parameters for parity tests: Xavier weights as init_flat, plus small random conv / fc1 biases
    (non-degenerate ReLU patterns), fc2 weights scaled by `fc2_gain` and an fc2 bias in +-`out_bias` px, so that |pred_h4p| is
    tens of pixels like a trained network's.  On Xavier weights alone pred_h4p is ~0.01 px and every pixel-unit tolerance is
    vacuous; with this recipe a relative error of 1e-5 in the regressor is 1e-3 px at the output."""
    specs = param_specs(patch_size)
    flat = init_flat(seed, patch_size)
    rng = np.random.default_rng(seed + 7919)
    for n, s in specs.items():
        if n.endswith("biases") and "fc2" not in n:
            flat[s.offset:s.offset + s.size] = rng.uniform(-bias_amp, bias_amp, size=s.size).astype(np.float32)
    s = specs["model/fc2/fc2/weights"]
    flat[s.offset:s.offset + s.size] *= np.float32(fc2_gain)
    s = specs["model/fc2/fc2/biases"]
    flat[s.offset:s.offset + s.size] = rng.uniform(-out_bias, out_bias, size=8).astype(np.float32)
    return flat


def unflatten(flat, specs=None):
    """Views (no copy) of a flat numpy / torch buffer, keyed by checkpoint name."""
    specs = specs or param_specs()
    return OrderedDict((n, flat[s.offset:s.offset + s.size].reshape(s.shape)) for n, s in specs.items())


def save_named_npz(path, flat, extra=None, patch_size=128):
    """Write the parameters under the reference's TF-Slim variable names and shapes (SURVEY §8f-2): a TF-1 checkpoint
    converts to / from this file with `{v.name[:-2]: sess.run(v) for v in tf.global_variables()}`."""
    flat = np.asarray(flat, dtype=np.float32)
    arrays = {n: np.array(v) for n, v in unflatten(flat, param_specs(patch_size)).items()}
    if extra:
        arrays.update(extra)
    np.savez(path, **arrays)


def load_named_npz(path, patch_size=128):
    """Inverse of save_named_npz: flat fp32 buffer in this package's layout (shapes are checked)."""
    specs = param_specs(patch_size)
    flat = np.zeros(total_floats(specs), dtype=np.float32)
    with np.load(path) as z:
        for n, s in specs.items():
            if n not in z:
                raise KeyError("checkpoint is missing variable %s" % n)
            a = np.asarray(z[n], dtype=np.float32)
            if tuple(a.shape) != s.shape:
                raise ValueError("variable %s has shape %s, expected %s" % (n, a.shape, s.shape))
            flat[s.offset:s.offset + s.size] = a.reshape(-1)
    return flat
