"""Burgess encoder (reference disvae/models/encoders.py:16-89) on the sm_90a kernels."""
from torch import nn

from disvae import ops
from disvae.utils.initialization import Conv4x4, Dense


def get_encoder(model_type):
    model_type = model_type.lower().capitalize()
    if model_type != "Burgess":
        raise ValueError("Unkown encoder: {}".format(model_type))
    return EncoderBurgess


class EncoderBurgess(nn.Module):
    """3 (32x32) or 4 (64x64) x [conv k4 s2 p1 -> ReLU] -> 512 -> 256 -> 256 -> 2*latent_dim.
    Same parameter names, shapes and creation order as the reference (encoders.py:54-67)."""

    def __init__(self, img_size, latent_dim=10):
        super().__init__()
        hid_channels, hidden_dim = 32, 256
        self.latent_dim = latent_dim
        self.img_size = img_size
        self.reshape = (hid_channels, 4, 4)
        n_chan = self.img_size[0]
        self.conv1 = Conv4x4(n_chan, hid_channels)
        self.conv2 = Conv4x4(hid_channels, hid_channels)
        self.conv3 = Conv4x4(hid_channels, hid_channels)
        if self.img_size[1] == self.img_size[2] == 64:
            self.conv_64 = Conv4x4(hid_channels, hid_channels)
        self.lin1 = Dense(hid_channels * 16, hidden_dim)
        self.lin2 = Dense(hidden_dim, hidden_dim)
        self.mu_logvar_gen = Dense(hidden_dim, self.latent_dim * 2)

    def _layers(self):
        convs = [self.conv1, self.conv2, self.conv3]
        if hasattr(self, "conv_64"):
            convs.append(self.conv_64)
        return convs, [self.lin1, self.lin2, self.mu_logvar_gen]

    def forward(self, x):
        if tuple(x.shape[1:]) != tuple(self.img_size):
            raise RuntimeError("expected images of shape {}, got {}".format(tuple(self.img_size), tuple(x.shape[1:])))
        convs, lins = self._layers()
        params = []
        for layer in convs + lins:
            params += [layer.weight, layer.bias]
        mu_logvar = ops.EncoderFn.apply(x, len(convs), *params)
        # interleaved split, encoders.py:86-87 (SURVEY.md trap T1)
        mu, logvar = mu_logvar.view(-1, self.latent_dim, 2).unbind(-1)
        return mu, logvar
