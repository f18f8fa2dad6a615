"""Write a video's frame files from its images and camera reconstruction (scripts/preprocess/davis/generate_frame_midas.py).

    python -m dvd_b200.prepare_frames --davis_root <DAVIS> --track <track> --midas_ckpt midas_cpkt.pt \
        --out <root>/frames_midas/<track> [--chunk 8]

Reads <DAVIS>/JPEGImages/1080p/<track>/*.jpg, Annotations/1080p/<track>/*.png and triangulation/<track>.{intrinsics.txt,
matrices.txt,obj}, runs MiDaS and the scale calibration on the GPU (dvd_b200.frames) and writes frame_%05d.npz under --out,
where prepare_pairs and the video_frames dataset read them.
"""
import argparse
import time

from .frames import FrameBuilder


def main(argv=None):
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument('--davis_root', required=True, help='directory holding JPEGImages/, Annotations/ and triangulation/')
    p.add_argument('--track', required=True, help='track name')
    p.add_argument('--midas_ckpt', required=True, help='MiDaS checkpoint (midas_cpkt.pt)')
    p.add_argument('--out', required=True, help='directory for frame_%%05d.npz')
    p.add_argument('--chunk', type=int, default=8, help='frames per device pass')
    a = p.parse_args(argv)
    import torch
    from .third_party.MiDaS import MidasNet
    t0 = time.time()
    net = MidasNet(a.midas_ckpt, non_negative=True, resize=[256, 512], normalize_input=True).cuda().eval()
    b = FrameBuilder(a.davis_root, a.track, net, chunk=a.chunk)
    n = b.write(a.out)
    torch.cuda.synchronize()
    print('%d frames of %s written to %s in %.1f s (scale %.6g)' % (n, a.track, a.out, time.time() - t0, b.scale))


if __name__ == '__main__':
    main()
