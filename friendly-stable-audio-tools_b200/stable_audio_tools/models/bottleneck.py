"""Bottlenecks on the hot path (reference ``models/bottleneck.py:10-115``).  The VAE
reparameterisation stays in PyTorch on purpose: it draws from the caller's torch RNG
(``randn_like``), and the kernel boundary is the deterministic ``mean | scale`` tensor
(SURVEY.md H8).  The Wasserstein and L2 bottlenecks are a few torch ops once per call, likewise."""
import torch
from torch import nn
from torch.nn import functional as F


class Bottleneck(nn.Module):
    def __init__(self, is_discrete: bool = False):
        super().__init__()
        self.is_discrete = is_discrete

    def encode(self, x, return_info=False, **kwargs):
        raise NotImplementedError

    def decode(self, x):
        raise NotImplementedError


class TanhBottleneck(Bottleneck):
    def encode(self, x, return_info=False):
        x = torch.tanh(x)
        return (x, {}) if return_info else x

    def decode(self, x):
        return x


def vae_sample(mean, scale):
    stdev = nn.functional.softplus(scale) + 1e-4
    var = stdev * stdev
    latents = torch.randn_like(mean) * stdev + mean
    kl = (mean * mean + var - torch.log(var) - 1).sum(1).mean()
    return latents, kl


class VAEBottleneck(Bottleneck):
    def encode(self, x, return_info=False, **kwargs):
        mean, scale = x.chunk(2, dim=1)
        z, kl = vae_sample(mean, scale)
        return (z, {"kl": kl}) if return_info else z

    def decode(self, x):
        return x


def compute_mean_kernel(x, y):
    kernel_input = (x[:, None] - y[None]).pow(2).mean(2) / x.shape[-1]
    return torch.exp(-kernel_input).mean()


def compute_mmd(latents):
    """Maximum mean discrepancy between the latent frames and as many standard-normal draws (reference :68-82)."""
    latents_reshaped = latents.permute(0, 2, 1).reshape(-1, latents.shape[1])
    noise = torch.randn_like(latents_reshaped)
    latents_kernel = compute_mean_kernel(latents_reshaped, latents_reshaped)
    noise_kernel = compute_mean_kernel(noise, noise)
    latents_noise_kernel = compute_mean_kernel(latents_reshaped, noise)
    return (latents_kernel + noise_kernel - 2 * latents_noise_kernel).mean()


class WassersteinBottleneck(Bottleneck):
    """Identity on encode (with the MMD loss in training); decode appends ``noise_augment_dim`` channels of standard
    normal noise, drawn on the CPU from the global torch RNG and moved to the input's device, as the reference does
    (:85-103), so a seeded decode draws the reference's noise."""

    def __init__(self, noise_augment_dim: int = 0):
        super().__init__(is_discrete=False)
        self.noise_augment_dim = noise_augment_dim

    def encode(self, x, return_info=False, **kwargs):
        info = {}
        if self.training and return_info:
            info["mmd"] = compute_mmd(x)
        return (x, info) if return_info else x

    def decode(self, x):
        if self.noise_augment_dim > 0:
            noise = torch.randn(x.shape[0], self.noise_augment_dim, x.shape[-1]).type_as(x)
            x = torch.cat([x, noise], dim=1)
        return x


class L2Bottleneck(Bottleneck):
    """Unit L2 norm over the channels on encode and on decode (reference :106-115)."""

    def encode(self, x, return_info=False, **kwargs):
        x = F.normalize(x, dim=1)
        return (x, {}) if return_info else x

    def decode(self, x):
        return F.normalize(x, dim=1)
