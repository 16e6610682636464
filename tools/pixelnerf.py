"""pixelNeRF from the command line (the reference's contrib/pixelnerf main.py):

    python tools/pixelnerf.py --data tiny_nerf_data.npz --task train [--epochs 100] [--save net.pth] [--pixel_aligned]
    python tools/pixelnerf.py --data tiny_nerf_data.npz --task test --ckpt net.pth
    python tools/pixelnerf.py --data tiny_nerf_data.npz --task video --ckpt net.pth [--out video.mp4]
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from jnerf_b200.pixelnerf_runner import PixelNeRFRunner, pixelnerf_cfg  # noqa: E402
from jnerf_b200.utils.config import get_cfg, update_cfg  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--data", required=True)
    ap.add_argument("--task", choices=["train", "test", "video"], default="train")
    ap.add_argument("--epochs", type=int, default=None)
    ap.add_argument("--ckpt", default=None, help="a .pth state dict to start from")
    ap.add_argument("--save", default=None, help="where train writes the .pth state dict")
    ap.add_argument("--out", default=None, help="the video path")
    ap.add_argument("--encoder_weights", default=None, help="a torchvision resnet34 state dict")
    ap.add_argument("--pixel_aligned", action="store_true")
    ap.add_argument("--log_dir", default="./logs")
    a = ap.parse_args()
    get_cfg().clear()
    over = dict(pixel_aligned=a.pixel_aligned, log_dir=a.log_dir, encoder_weights=a.encoder_weights)
    if a.epochs is not None:
        over["epoch"] = a.epochs
    update_cfg(**pixelnerf_cfg(a.data, **over))
    r = PixelNeRFRunner()
    if a.ckpt:
        r.load_ckpt(a.ckpt)
    if a.task == "train":
        r.train(log_every=14)
        if a.save:
            r.save_ckpt(a.save)
        r.test()
    elif a.task == "test":
        r.test()
    else:
        print(r.render(a.out))


if __name__ == "__main__":
    main()
