"""Parameter holders of G-SphereNet's flow layers and focus classifier (reference
dig/ggraph3D/method/G_SphereNet/model/net_utils.py).  Their arithmetic during generation is in sphgen.py's step, on the
sm_90a kernels (flow reverse: dig3d_gsphere_flow_reverse), and during training in sphgen.py's forward
(dig3d_gsphere_flow_fwd / _bwd)."""
import torch
import torch.nn as nn


def _training_not_built(what):
    raise NotImplementedError(f"{what}: the flow and focus layers run inside SphGen.forward / SphGen.generate on the "
                              "GPU kernels, not as separate modules (DESIGN.md section 6)")


class Rescale(nn.Module):
    def __init__(self):
        super().__init__()
        self.weight = nn.Parameter(torch.zeros([1]))

    def forward(self, x):
        _training_not_built("Rescale.forward")


class ST_Net_Exp(nn.Module):
    """linear2(tanh(linear1(x))) -> (s = exp(rescale) * tanh(s), t)   (net_utils.py:5-37)."""

    def __init__(self, input_dim, output_dim, hid_dim=64, num_layers=2, bias=True):
        super().__init__()
        self.num_layers = num_layers
        self.input_dim, self.hid_dim, self.output_dim, self.bias = input_dim, hid_dim, output_dim, bias
        self.linear1 = nn.Linear(input_dim, hid_dim, bias=bias)
        self.linear2 = nn.Linear(hid_dim, output_dim * 2, bias=bias)
        self.rescale1 = Rescale()
        self.tanh = nn.Tanh()
        self.reset_parameters()

    def reset_parameters(self):
        nn.init.xavier_uniform_(self.linear1.weight)
        nn.init.constant_(self.linear2.weight, 1e-10)
        if self.bias:
            nn.init.constant_(self.linear1.bias, 0.)
            nn.init.constant_(self.linear2.bias, 0.)

    def forward(self, x):
        _training_not_built("ST_Net_Exp.forward")


def init_layer(layer, w_scale=1.0):
    torch.nn.init.orthogonal_(layer.weight.data)
    layer.weight.data.mul_(w_scale)
    torch.nn.init.constant_(layer.bias.data, 0)
    return layer


class MLP(nn.Module):
    """Focus classifier sigmoid(lin(relu(lin(x))))   (net_utils.py:61-72)."""

    def __init__(self, input_dim, hidden_units=128):
        super().__init__()
        self.layers = nn.Sequential(init_layer(nn.Linear(input_dim, hidden_units)), nn.ReLU(),
                                    init_layer(nn.Linear(hidden_units, 1)), nn.Sigmoid())

    def forward(self, x):
        _training_not_built("MLP.forward")
