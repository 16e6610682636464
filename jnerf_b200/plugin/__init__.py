"""Host-side mirror of JNeRF's plugin interface for the Instant-NGP and vanilla NeRF paths (registered under the same names)."""
from . import encoders, network, nerf, sampler, losses, optim, dataset  # noqa: F401  (registration side effects)
