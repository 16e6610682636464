"""The pixelNeRF operators of jnerf_b200/ops.py (pixelnerf_fwd / pixelnerf_bwd / pixelnerf_composite_fwd / pixelnerf_composite_loss_bwd)
restated in float64 torch from the reference's Network.py, Render.py and Dataset.py (through plugin/pixelnerf.py's restatement), installed
over jnerf_b200.ops on top of tests/cpu_backend.py so that PixelNeRFRunner's host logic runs without a GPU."""
import torch


def install(monkeypatch):
    import cpu_backend
    import jnerf_b200.ops as real_ops
    from jnerf_b200.plugin import pixelnerf as pn
    fake = cpu_backend.install(monkeypatch)

    def raw64(rays, z, params, feats, cams, scale, pixel_aligned, state=None):
        state = pn.unpack(params.double()) if state is None else state
        state = {k: v.double() for k, v in state.items()}
        S = z.shape[0]
        pts = (rays[:, None, :3].double() + rays[:, None, 3:6].double() * z[None, :, None].double()).reshape(-1, 3)
        enc = pn.positional_encoding(pts, rays[:, None, 3:6].double().expand(-1, S, -1).reshape(-1, 3))
        feat = pn.feature_matching(feats.double(), pts, cams.double(), scale, pixel_aligned)
        return pn.network_torch(state, enc, feat, torch.float64)

    def pixelnerf_workspace_bytes(n_rows, n_ref):
        return 1, 1, 1

    def pixelnerf_fwd(rays, z, params, feats, cams, scale, pixel_aligned=False, saved=None, scratch=None, out=None):
        fake._log("pixelnerf_fwd")
        if saved is not None:
            fake.pixelnerf_saved = (rays.clone(), z.clone(), cams, float(scale), bool(pixel_aligned))
        raw = raw64(rays, z, params, feats, cams, scale, pixel_aligned).half()
        if out is not None:
            out.copy_(raw)
            return out
        return raw

    def pixelnerf_bwd(rays_count, n_samples, params, feats, saved, raw, draw, scratch=None):
        fake._log("pixelnerf_bwd")
        rays, z, cams, scale, aligned = fake.pixelnerf_saved
        assert rays.shape[0] == rays_count and z.shape[0] == n_samples
        state = {k: v.double().requires_grad_() for k, v in pn.unpack(params).items()}
        with torch.enable_grad():
            (raw64(rays, z, params, feats, cams, scale, aligned, state) * draw.double()).sum().backward()
        return pn.pack({k: v.grad for k, v in state.items()}).float()

    def pixelnerf_composite_fwd(raw, z, rays):
        fake._log("pixelnerf_composite_fwd")
        return tuple(t.float() for t in pn.composite_torch(raw.double(), z.double(), rays.double()))

    def pixelnerf_composite_loss_bwd(raw, z, rays, target, grad_scale=1.0):
        fake._log("pixelnerf_composite_loss_bwd")
        r = raw.double().requires_grad_()
        with torch.enable_grad():
            rgb = pn.composite_torch(r, z.double(), rays.double())[0]
            per_ray = ((rgb - target.double()) ** 2).sum(-1) / (3 * rays.shape[0])
            (per_ray.sum() * grad_scale).backward()
        return rgb.detach().float(), per_ray.detach().float(), r.grad.clamp(-65504, 65504).to(raw.dtype)

    for name, fn in (("pixelnerf_workspace_bytes", pixelnerf_workspace_bytes), ("pixelnerf_fwd", pixelnerf_fwd), ("pixelnerf_bwd", pixelnerf_bwd),
                     ("pixelnerf_composite_fwd", pixelnerf_composite_fwd), ("pixelnerf_composite_loss_bwd", pixelnerf_composite_loss_bwd)):
        monkeypatch.setattr(real_ops, name, fn)
    return fake
