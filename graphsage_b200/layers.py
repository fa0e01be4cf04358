"""Layer base and Dense - the API shell of reference graphsage/layers.py:28-116 over the
library's CUDA kernels (Dense is only used as the max-pool aggregator's MLP)."""
import torch

from . import ops
from .inits import glorot, zeros

_LAYER_UIDS = {}


def get_layer_uid(layer_name=""):
    """reference graphsage/layers.py:19-26."""
    _LAYER_UIDS[layer_name] = _LAYER_UIDS.get(layer_name, 0) + 1
    return _LAYER_UIDS[layer_name]


def relu(x):
    """Stand-in for tf.nn.relu as the `act` argument; recognised and fused into the GEMM epilogue."""
    return torch.relu(x)


def identity(x):
    return x


def act_code(act):
    """(fused activation code, python callable still to apply)."""
    if act is relu or act is torch.relu or act is torch.nn.functional.relu:
        return ops.ACT_RELU, None
    if act is None or act is identity:
        return ops.ACT_NONE, None
    return ops.ACT_NONE, act            # arbitrary callable (e.g. the reference's `lambda x: x`): applied after


class Layer(object):
    """reference graphsage/layers.py:28-70: kwarg whitelist, auto name `<class>_<uid>`, .vars dict,
    __call__ -> _call."""

    ALLOWED_KWARGS = frozenset(("name", "logging", "model_size"))

    def __init__(self, **kwargs):
        unknown = [k for k in kwargs if k not in self.ALLOWED_KWARGS]
        assert not unknown, "Invalid keyword argument: " + unknown[0]
        self.vars, self.sparse_inputs = {}, False
        self.logging = bool(kwargs.get("logging", False))
        self.name = kwargs.get("name") or self._auto_name()

    @classmethod
    def _auto_name(cls):
        kind = cls.__name__.lower()
        return "%s_%d" % (kind, get_layer_uid(kind))

    def _call(self, inputs):
        return inputs

    def __call__(self, inputs):
        return self._call(inputs)

    def parameters(self):
        return list(self.vars.values())


class Dense(Layer):
    """act(dropout(x) @ W + b) - reference graphsage/layers.py:73-116 (xavier-uniform W, zero bias)."""

    def __init__(self, input_dim, output_dim, dropout=0., act=relu, placeholders=None, bias=True, featureless=False,
                 sparse_inputs=False, device="cuda", math=ops.MATH_FP32_SIMT, **kwargs):
        super(Dense, self).__init__(**kwargs)
        if sparse_inputs:
            raise NotImplementedError("sparse_inputs is not on the hot path")
        self.dropout = dropout
        self.act = act
        self.featureless = featureless
        self.bias = bias
        self.input_dim = input_dim
        self.output_dim = output_dim
        self.math = math
        self.vars["weights"] = glorot((input_dim, output_dim), name="weights", device=device)
        if self.bias:
            self.vars["bias"] = zeros((output_dim,), name="bias", device=device)

    def _call(self, inputs):
        x = inputs
        if self.dropout:
            x = torch.nn.functional.dropout(x, p=float(self.dropout), training=True)
        code, post = act_code(self.act)
        if getattr(self, "_packed", None) is None:
            self._packed = ops.PackedWeights()
        y = ops.sage_gemm([(x, self.input_dim, self.vars["weights"])], bias=self.vars.get("bias"), act=code,
                          math=self.math, packed=self._packed)
        return post(y) if post else y
