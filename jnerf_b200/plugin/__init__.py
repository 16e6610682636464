"""Host-side mirror of JNeRF's plugin interface for the Instant-NGP, vanilla NeRF, Mip-NeRF and Plenoxels paths (registered under the same names)."""
from . import encoders, network, nerf, sampler, losses, optim, dataset, mip, svox2  # noqa: F401  (registration side effects)
