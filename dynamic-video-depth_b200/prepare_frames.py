"""Write a video's frame files from its images and camera reconstruction (scripts/preprocess/{davis,shutterstock}/
generate_frame_midas.py).

    python -m dvd_b200.prepare_frames --davis_root <DAVIS> --track <track> --midas_ckpt midas_cpkt.pt \
        --out <root>/frames_midas/<track> [--chunk 8]
    python -m dvd_b200.prepare_frames --shutterstock_root <SS> [--track <track>] --midas_ckpt midas_cpkt.pt \
        --out <root>/frames_midas [--chunk 8]
    python -m dvd_b200.prepare_frames --colmap_model <sparse/0> --images <images> [--masks <masks>] \
        --midas_ckpt midas_cpkt.pt --out <root>/frames_midas/<track> [--chunk 8]

DAVIS: reads <DAVIS>/JPEGImages/1080p/<track>/*.jpg, Annotations/1080p/<track>/*.png and triangulation/<track>.{intrinsics.txt,
matrices.txt,obj}, runs MiDaS and the scale calibration on the GPU (dvd_b200.frames) and writes frame_%05d.npz under --out,
where prepare_pairs and the video_frames dataset read them.

ShutterStock: reads the per-frame HDF5 files <SS>/triangulation/<track>/*.h5 (h5py) of every track, or of --track alone, runs
MiDaS at the stored size and the dense scale calibration on the GPU, and writes <out>/<track>/frame_%05d.npz, where
prepare_pairs and the shutterstock dataset (--track_id, the track's index in the sorted list) read them. A track whose
frame 0 camera matrix has fewer than 3 rows is skipped, as the reference skips it.

COLMAP: reads a sparse model (cameras, images, points3D, as .bin or .txt) with one PINHOLE or SIMPLE_PINHOLE camera, the
registered images under --images and, optionally, motion masks <masks>/<image name without extension>.png (all zero when
--masks is omitted), and writes the DAVIS frame files of the registered images in the sorted order of their names under --out.
Every image file under --images must be registered in the model.
"""
import argparse
import os
import time

from .frames import ColmapFrameBuilder, FrameBuilder, ShutterstockFrameBuilder, read_shutterstock_track, shutterstock_tracks


def main(argv=None):
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    src = p.add_mutually_exclusive_group(required=True)
    src.add_argument('--davis_root', help='directory holding JPEGImages/, Annotations/ and triangulation/')
    src.add_argument('--shutterstock_root', help='directory holding triangulation/<track>/*.h5')
    src.add_argument('--colmap_model', help='COLMAP sparse model directory (cameras, images, points3D as .bin or .txt)')
    p.add_argument('--images', default=None, help='with --colmap_model: directory of the registered images')
    p.add_argument('--masks', default=None, help='with --colmap_model: directory of <image stem>.png motion masks (optional)')
    p.add_argument('--track', default=None, help='track name (required with --davis_root; every track when omitted with '
                                                 '--shutterstock_root)')
    p.add_argument('--midas_ckpt', required=True, help='MiDaS checkpoint (midas_cpkt.pt)')
    p.add_argument('--out', required=True, help='directory for frame_%%05d.npz (with --shutterstock_root: for <track>/frame_%%05d.npz)')
    p.add_argument('--chunk', type=int, default=8, help='frames per device pass')
    a = p.parse_args(argv)
    if a.davis_root is not None and a.track is None:
        p.error('--davis_root needs --track')
    if a.colmap_model is not None and a.images is None:
        p.error('--colmap_model needs --images')
    if a.colmap_model is None and (a.images is not None or a.masks is not None):
        p.error('--images and --masks go with --colmap_model')
    if a.colmap_model is not None and a.track is not None:
        p.error('--track does not go with --colmap_model: --out names the video')
    import torch
    from .third_party.MiDaS import MidasNet
    t0 = time.time()
    if a.davis_root is not None:
        net = MidasNet(a.midas_ckpt, non_negative=True, resize=[256, 512], normalize_input=True).cuda().eval()
        b = FrameBuilder(a.davis_root, a.track, net, chunk=a.chunk)
        n = b.write(a.out)
        torch.cuda.synchronize()
        print('%d frames of %s written to %s in %.1f s (scale %.6g)' % (n, a.track, a.out, time.time() - t0, b.scale))
        return
    if a.colmap_model is not None:
        net = MidasNet(a.midas_ckpt, non_negative=True, resize=[256, 512], normalize_input=True).cuda().eval()
        b = ColmapFrameBuilder(a.images, a.colmap_model, net, masks_dir=a.masks, chunk=a.chunk)
        n = b.write(a.out)
        torch.cuda.synchronize()
        print('%d frames of %s written to %s in %.1f s (scale %.6g)' % (n, a.colmap_model, a.out, time.time() - t0, b.scale))
        return
    names = [os.path.basename(t) for t in shutterstock_tracks(a.shutterstock_root)]
    if a.track is not None and a.track not in names:
        p.error('no track %s under %s' % (a.track, os.path.join(a.shutterstock_root, 'triangulation')))
    net = MidasNet(a.midas_ckpt, non_negative=True, resize=None, normalize_input=True).cuda().eval()
    for tid, name in enumerate(names):
        if a.track is not None and name != a.track:
            continue
        t1 = time.time()
        _, handles = read_shutterstock_track(a.shutterstock_root, tid)
        if handles is None:
            print('track %d (%s) skipped: its first camera matrix has fewer than 3 rows' % (tid, name))
            continue
        try:
            b = ShutterstockFrameBuilder(handles, net, chunk=a.chunk)
            n = b.write(os.path.join(a.out, name))
        finally:
            for h in handles:
                h.close()
        torch.cuda.synchronize()
        print('track %d: %d frames of %s written to %s in %.1f s (scale %.6g)' % (tid, n, name, os.path.join(a.out, name),
                                                                                 time.time() - t1, b.scale))


if __name__ == '__main__':
    main()
