"""Host-side mirror of JNeRF's plugin interface for the Instant-NGP, vanilla NeRF and Mip-NeRF paths (registered under the same names)."""
from . import encoders, network, nerf, sampler, losses, optim, dataset, mip  # noqa: F401  (registration side effects)
