"""VAE wrapper (reference disvae/models/vae.py:12-101)."""
import torch
from torch import nn

from disvae import ops
from disvae.utils.initialization import weights_init
from .decoders import get_decoder
from .encoders import get_encoder

MODELS = ["Burgess"]


def init_specific_model(model_type, img_size, latent_dim):
    """Return a VAE with encoder and decoder of `model_type` (vae.py:15-26)."""
    model_type = model_type.lower().capitalize()
    if model_type not in MODELS:
        err = "Unkown model_type={}. Possible values: {}"
        raise ValueError(err.format(model_type, MODELS))
    model = VAE(img_size, get_encoder(model_type), get_decoder(model_type), latent_dim)
    model.model_type = model_type
    return model


def noise_key(seed, salt=0):
    """Philox key of the reparameterisation noise of a process seeded with `seed` (`salt`: parallel.rank_salt())."""
    return (int(seed) + salt) & 0xFFFFFFFFFFFFFFFF


class VAE(nn.Module):
    def __init__(self, img_size, encoder, decoder, latent_dim):
        super().__init__()
        if list(img_size[1:]) not in [[32, 32], [64, 64]]:
            raise RuntimeError("{} sized images not supported. Only (None, 32, 32) and (None, 64, 64) supported. "
                               "Build your own architecture or reshape images!".format(img_size))
        self.latent_dim = latent_dim
        self.img_size = img_size
        self.num_pixels = self.img_size[1] * self.img_size[2]
        self.encoder = encoder(img_size, self.latent_dim)
        self.decoder = decoder(img_size, self.latent_dim)
        self._rng_seed = None          # Philox key, fixed at first use from torch.initial_seed()
        self._rng_offset = None        # device-side Philox counter (uint64 in an int64 tensor)
        self._eps_queue = []           # injected noise (parity tests), consumed FIFO
        self.reset_parameters()

    # -- device noise stream ------------------------------------------------------------
    def _noise_state(self, device):
        if self._rng_offset is None or self._rng_offset.device != device:
            from disvae.parallel import rank_salt
            # identically seeded replicas (main.py's set_seed) must still draw different noise for their shards
            self.seed_noise(noise_key(torch.initial_seed(), rank_salt()), device)
        return self._rng_seed, self._rng_offset

    def seed_noise(self, key, device):
        """Fix the Philox key of the reparameterisation noise (what the first training step would take from
        torch.initial_seed(); noise_key) and start its counter at 0 on `device`."""
        self._rng_seed = int(key)
        self._rng_offset = torch.zeros(1, dtype=torch.int64, device=device)

    def reparameterize(self, mean, logvar, eps=None):
        """vae.py:52-71.  Training: mean + exp(0.5*logvar) * eps with eps ~ N(0,1) drawn on the
        device (Philox4x32-10) unless `eps` is given; eval: the mean."""
        if self.training:
            if eps is None and self._eps_queue:
                eps = self._eps_queue.pop(0).to(mean.device)
            seed, off = (0, None) if eps is not None else self._noise_state(mean.device)
            return ops.ReparamFn.apply(mean, logvar, eps, seed, off)
        return mean

    def inject_noise(self, eps_list):
        """Queue eps tensors ([B, latent_dim]) to be used by the next reparameterize calls
        instead of device-generated noise (deterministic parity runs)."""
        self._eps_queue = list(eps_list)

    def forward(self, x, eps=None):
        """vae.py:73-85: (reconstruction, (mean, logvar), latent sample)."""
        latent_dist = self.encoder(x)
        latent_sample = self.reparameterize(*latent_dist, eps=eps)
        reconstruct = self.decoder(latent_sample)
        return reconstruct, latent_dist, latent_sample

    def reset_parameters(self):
        self.apply(weights_init)

    def sample_latent(self, x, eps=None):
        """vae.py:90-101"""
        latent_dist = self.encoder(x)
        return self.reparameterize(*latent_dist, eps=eps)
