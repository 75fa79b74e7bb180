"""Burgess decoder (reference disvae/models/decoders.py:16-84) on the sm_90a kernels."""
from torch import nn

from disvae import ops
from disvae.utils.initialization import ConvT4x4, Dense


def get_decoder(model_type):
    model_type = model_type.lower().capitalize()
    if model_type != "Burgess":
        raise ValueError("Unkown decoder: {}".format(model_type))
    return DecoderBurgess


class DecoderBurgess(nn.Module):
    """latent -> 256 -> 256 -> 512 -> view(32,4,4) -> 3/4 x convT k4 s2 p1 (+ReLU), sigmoid last.
    Same parameter names, shapes and creation order as the reference (decoders.py:53-65)."""

    def __init__(self, img_size, latent_dim=10):
        super().__init__()
        hid_channels, hidden_dim = 32, 256
        self.img_size = img_size
        self.reshape = (hid_channels, 4, 4)
        n_chan = self.img_size[0]
        self.lin1 = Dense(latent_dim, hidden_dim)
        self.lin2 = Dense(hidden_dim, hidden_dim)
        self.lin3 = Dense(hidden_dim, hid_channels * 16)
        if self.img_size[1] == self.img_size[2] == 64:
            self.convT_64 = ConvT4x4(hid_channels, hid_channels)
        self.convT1 = ConvT4x4(hid_channels, hid_channels)
        self.convT2 = ConvT4x4(hid_channels, hid_channels)
        self.convT3 = ConvT4x4(hid_channels, n_chan)

    def _layers(self):
        convTs = [self.convT_64] if hasattr(self, "convT_64") else []
        convTs += [self.convT1, self.convT2, self.convT3]
        return [self.lin1, self.lin2, self.lin3], convTs

    def forward(self, z):
        lins, convTs = self._layers()
        params = []
        for layer in lins + convTs:
            params += [layer.weight, layer.bias]
        return ops.DecoderFn.apply(z, len(convTs), self.img_size[0], *params)
