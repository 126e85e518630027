"""Parameter containers for the NICE decoders.

The fused kernels consume the decoders' parameter tensors directly (by device pointer); they accept the
reference's own `NICE` module (src/conv_onet/models/decoder.py:277-342) unchanged.  `NICEDecoders` is a
stand-alone container with the SAME module tree / state_dict keys (embedder._B, pts_linears.i.{weight,bias},
fc_c.i.{weight,bias}, output_linear.{weight,bias}), so checkpoints are interchangeable, for use where the
reference package is not importable.  It holds parameters only; evaluation always goes through the CUDA path.
"""
import torch
import torch.nn as nn

from . import _lib
from ._lib import LEVELS

HIDDEN, EMBED, C_DIM = 32, 93, 32


def _xavier_linear(n_in, n_out, gain, reference_draws=False):
    """reference_draws: draw only xavier's uniforms, as DenseLayer (whose reset_parameters replaces nn.Linear's) does; otherwise
    nn.Linear's own kaiming and bias draws come first."""
    lin = nn.utils.skip_init(nn.Linear, n_in, n_out) if reference_draws else nn.Linear(n_in, n_out)
    nn.init.xavier_uniform_(lin.weight, gain=gain)      # DenseLayer.reset_parameters, decoder.py:77-82
    nn.init.zeros_(lin.bias)
    return lin


class _Embedder(nn.Module):
    def __init__(self, scale=25.0):
        super().__init__()
        self._B = nn.Parameter(torch.randn(3, EMBED) * scale)     # decoder.py:21-22


class DecoderMLP(nn.Module):
    """Parameters of MLP (xyz=True; middle/fine/color) or MLP_no_xyz (xyz=False; coarse)."""

    def __init__(self, name, xyz=True, c_dim=C_DIM, color=False, reference_draws=False):
        super().__init__()
        self.name, self.xyz, self.c_dim, self.color = name, xyz, c_dim, color
        relu_gain = nn.init.calculate_gain("relu")
        if xyz:
            self.fc_c = nn.ModuleList([nn.Linear(c_dim, HIDDEN) for _ in range(5)])
            self.embedder = _Embedder()
            ins = [EMBED, HIDDEN, HIDDEN, HIDDEN + EMBED, HIDDEN]
        else:
            ins = [HIDDEN, HIDDEN, HIDDEN, HIDDEN + c_dim, HIDDEN]
        self.pts_linears = nn.ModuleList([_xavier_linear(i, HIDDEN, relu_gain, reference_draws) for i in ins])
        self.output_linear = _xavier_linear(HIDDEN, 4 if color else 1, 1.0, reference_draws)


class NICEDecoders(nn.Module):
    def __init__(self, coarse=True, reference_draws=False):
        """reference_draws: draw from torch's global generator exactly as config.get_model(cfg, nice=True) does (fc_c as nn.Linear, the
        embedder's randn, then xavier only for pts_linears and output_linear; coarse, middle, fine, colour), so that under one seed the
        parameters come out bit-identical to the reference's.  The default keeps this class's own draws."""
        super().__init__()
        r = reference_draws
        if coarse:
            self.coarse_decoder = DecoderMLP("coarse", xyz=False, reference_draws=r)
        self.middle_decoder = DecoderMLP("middle", reference_draws=r)
        self.fine_decoder = DecoderMLP("fine", c_dim=2 * C_DIM, reference_draws=r)
        self.color_decoder = DecoderMLP("color", color=True, reference_draws=r)

    @classmethod
    def from_state(cls, state, device=None):
        """state: {'coarse'|'middle'|'fine'|'color': {param name: tensor}} (oracle.torch_port.decoders_state format)."""
        m = cls(coarse="coarse" in state)
        with torch.no_grad():
            for lvl, sd in state.items():
                getattr(m, lvl + "_decoder").load_state_dict({k: v.detach().clone() for k, v in sd.items()})
        return m.to(device) if device is not None else m


def decoder_module(decoders, level_name):
    sub = getattr(decoders, level_name + "_decoder", None)
    if sub is None:
        raise RuntimeError("decoders object has no %s_decoder" % level_name)
    return sub


def named_params(decoders, level_name):
    """{reference parameter name: tensor} of one decoder, whatever module class holds it."""
    sub = decoder_module(decoders, level_name)
    out = dict(sub.named_parameters())
    for k, v in sub.named_buffers():
        out.setdefault(k, v)
    if "embedder._B" not in out and hasattr(sub, "embedder") and hasattr(sub.embedder, "_B"):
        out["embedder._B"] = sub.embedder._B          # non-learnable variant keeps _B as a plain tensor
    return out


def decoder_params_struct(decoders, level_name):
    """nsb_decoder_params of one decoder (pointers into the live nn.Parameters)."""
    p = named_params(decoders, level_name)
    li = LEVELS.index(level_name)
    dp = _lib.DecoderParams()
    for t in p.values():
        if not t.is_cuda or t.dtype != torch.float32 or not t.is_contiguous():
            raise RuntimeError("nice_slam_b200: decoder parameters must be contiguous float32 CUDA tensors")
    if li != 0:
        dp.B = p["embedder._B"].data_ptr()
    for i in range(5):
        dp.W[i] = p["pts_linears.%d.weight" % i].data_ptr()
        dp.b[i] = p["pts_linears.%d.bias" % i].data_ptr()
        if li != 0:
            dp.Wc[i] = p["fc_c.%d.weight" % i].data_ptr()
            dp.bc[i] = p["fc_c.%d.bias" % i].data_ptr()
    dp.Wo = p["output_linear.weight"].data_ptr()
    dp.bo = p["output_linear.bias"].data_ptr()
    return dp
