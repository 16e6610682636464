"""NerfRunner: the Runner for vanilla NeRF (OriginNeRFNetworks, projects/nerf/configs/nerf_base.py) with the two reference tools that
Runner itself refuses for this model: mesh extraction (tools/extract_mesh.py; the density lattice on the fp16 kernels,
ngp_nerf_density_lattice, DESIGN.md section 4) and the params.pkl interchange (runner/runner.py:123-151; the 24 tensors under the
reference's names, utils/ckpt_compat.py).  Training, rendering and the .pt checkpoint are Runner's."""
import numpy as np

from .plugin.nerf import OriginNeRFNetworks
from .runner import Runner
from .utils import ckpt_compat as cc


class NerfRunner(Runner):
    def __init__(self, rank=0, world_size=1, process_group=None):
        super().__init__(rank, world_size, process_group)
        if not isinstance(self.model, OriginNeRFNetworks):
            raise ValueError(f"NerfRunner runs OriginNeRFNetworks (vanilla NeRF); the config builds {type(self.model).__name__}: use Runner")

    def _density_lattice_fn(self):
        return self.model.density_lattice

    def extract_mesh(self, out_dir, resolution=512, mcube_smooth=False):
        """Runner.extract_mesh with the lattice of the fp16 NeRF kernels; the colour rays go through model.infer."""
        if not self.model.using_fp16:
            raise NotImplementedError("extract_mesh: the density lattice of OriginNeRFNetworks runs on the fused kernels (fp16=True)")
        return super().extract_mesh(out_dir, resolution, mcube_smooth)

    def _to_reference(self, ck, adam_hyper, expdecay_hyper):
        return cc.nerf_native_to_reference(ck, adam_hyper=adam_hyper, expdecay_hyper=expdecay_hyper,
                                           param_dtype=np.float16 if self.model.using_fp16 else np.float32)

    def _from_reference_file(self, path):
        return cc.load_native_from_reference_file(path, None, "cuda", {k: v.dtype for k, v in self.model.state_dict().items()},
                                                  nerf_fp16=self.model.using_fp16)
