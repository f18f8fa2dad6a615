"""CPU: dvd_b200.frames.read_colmap_model on COLMAP sparse models written here in both of COLMAP's forms (the layout of its
read_write_model.py, little-endian), the checks ColmapFrameBuilder makes before it touches the GPU, and a scene written twice,
as a DAVIS track and as a COLMAP model over the same image files, whose cameras the two readers must return alike."""
import os
import struct

import numpy as np
import pytest
from PIL import Image

# COLMAP's camera models: id -> (name, parameter count)
MODELS = {0: ('SIMPLE_PINHOLE', 3), 1: ('PINHOLE', 4), 2: ('SIMPLE_RADIAL', 4), 3: ('RADIAL', 5), 4: ('OPENCV', 8),
          5: ('OPENCV_FISHEYE', 8), 6: ('FULL_OPENCV', 12), 7: ('FOV', 5), 8: ('SIMPLE_RADIAL_FISHEYE', 4),
          9: ('RADIAL_FISHEYE', 5), 10: ('THIN_PRISM_FISHEYE', 12)}
FLIP = np.diag([1.0, -1.0, -1.0, 1.0])
# unit quaternions (w, x, y, z) whose qvec2rotmat is exact: every entry 0 or +-1
EXACT_Q = [(1.0, 0.0, 0.0, 0.0), (0.5, 0.5, 0.5, 0.5), (0.0, 0.0, 0.0, 1.0), (0.5, -0.5, 0.5, -0.5), (0.0, 1.0, 0.0, 0.0),
           (0.5, 0.5, -0.5, 0.5), (0.0, 0.0, 1.0, 0.0), (0.5, -0.5, -0.5, -0.5)]
H, W = 160, 416
FX, FY, CX, CY = 256.0, 264.0, 207.5, 79.5               # DAVIS-side intrinsics: dyadic, so cx + 0.5 - 0.5 is exact


# ---- writers: COLMAP's two forms ----------------------------------------------------------------------------------------------
def write_bin(d, cameras, images, points):
    """cameras [(id, model id, width, height, params)], images [(id, qvec, tvec, camera id, name, [(x, y, point3D id)])],
    points [(id, xyz, rgb, error, [(image id, point2D index)])]"""
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, 'cameras.bin'), 'wb') as f:
        f.write(struct.pack('<Q', len(cameras)))
        for cid, model, w, h, params in cameras:
            f.write(struct.pack('<iiQQ', cid, model, w, h) + struct.pack('<%dd' % len(params), *params))
    with open(os.path.join(d, 'images.bin'), 'wb') as f:
        f.write(struct.pack('<Q', len(images)))
        for iid, q, t, cid, name, p2d in images:
            f.write(struct.pack('<i7di', iid, *q, *t, cid) + name.encode() + b'\0' + struct.pack('<Q', len(p2d)))
            for x, y, pid in p2d:
                f.write(struct.pack('<ddq', x, y, pid))
    with open(os.path.join(d, 'points3D.bin'), 'wb') as f:
        f.write(struct.pack('<Q', len(points)))
        for pid, xyz, rgb, err, track in points:
            f.write(struct.pack('<Q3d3BdQ', pid, *xyz, *rgb, err, len(track)))
            for iid, idx in track:
                f.write(struct.pack('<ii', iid, idx))


def write_txt(d, cameras, images, points):
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, 'cameras.txt'), 'w') as f:
        f.write('# Camera list with one line of data per camera:\n#   CAMERA_ID, MODEL, WIDTH, HEIGHT, PARAMS[]\n')
        for cid, model, w, h, params in cameras:
            f.write('%d %s %d %d %s\n' % (cid, MODELS[model][0], w, h, ' '.join(repr(float(p)) for p in params)))
    with open(os.path.join(d, 'images.txt'), 'w') as f:
        f.write('# Image list with two lines of data per image:\n')
        for iid, q, t, cid, name, p2d in images:
            f.write('%d %s %d %s\n' % (iid, ' '.join(repr(float(v)) for v in tuple(q) + tuple(t)), cid, name))
            f.write(' '.join('%r %r %d' % (float(x), float(y), pid) for x, y, pid in p2d) + '\n')
    with open(os.path.join(d, 'points3D.txt'), 'w') as f:
        f.write('# 3D point list with one line of data per point:\n')
        for pid, xyz, rgb, err, track in points:
            f.write('%d %s %d %d %d %r %s\n' % (pid, ' '.join(repr(float(v)) for v in xyz), *rgb, float(err),
                                                 ' '.join('%d %d' % tr for tr in track)))


# ---- a scene --------------------------------------------------------------------------------------------------------------
def scene(n=4, V=3000, exact=True, seed=0):
    """-> dict(cameras, images, points, w2c [n,4,4] by frame, xyz [V,3] by point id). Frame f is the image '%05d.jpg' % f. The
    images and points are listed in shuffled orders under shuffled ids; an unused OPENCV and an unused THIN_PRISM_FISHEYE
    camera come before the PINHOLE camera the images use. exact: rotations of EXACT_Q and dyadic translations, else
    general unit quaternions and translations."""
    g = np.random.default_rng(seed)
    if exact:
        qs = [EXACT_Q[f % len(EXACT_Q)] for f in range(n)]
        ts = [(0.25 * f - 0.5, 0.125 * (f % 3) - 0.125, 4.0 + 0.5 * (f % 2)) for f in range(n)]
    else:
        qs = [tuple(q / np.linalg.norm(q)) for q in g.normal(size=(n, 4)) * [4, 1, 1, 1]]
        ts = [tuple(v) for v in g.uniform(-0.3, 0.3, (n, 3)) + [0, 0, 4.1]]
    w2c = np.zeros((n, 4, 4))
    for f in range(n):
        w2c[f, :3, :3] = rotmat(qs[f])
        w2c[f, :3, 3] = ts[f]
        w2c[f, 3, 3] = 1
    cameras = [(7, 4, W, H, list(g.normal(size=8))), (9, 10, 2 * W, H, list(g.normal(size=12))),
               (3, 1, W, H, [FX, FY, CX + 0.5, CY + 0.5])]
    image_ids = g.permutation(np.arange(10, 10 + 3 * n, 3))
    images = [(int(image_ids[f]), qs[f], ts[f], 3, '%05d.jpg' % f, [(1.5, 2.5, -1), (3.25, 4.0, 17)] if f % 2 else [])
              for f in g.permutation(n)]
    xyz = g.uniform(-1, 1, (V, 3))
    point_ids = np.sort(g.choice(10 * V, V, replace=False)) + 1
    points = [(int(point_ids[v]), tuple(xyz[v]), tuple(int(c) for c in g.integers(0, 256, 3)), float(g.random()),
               [(int(image_ids[0]), v % 5), (int(image_ids[-1]), v % 7)][: v % 3]) for v in g.permutation(V)]
    return dict(cameras=cameras, images=images, points=points, w2c=w2c, xyz=xyz, n=n)


def rotmat(q):
    """qvec2rotmat written out (COLMAP's expressions)"""
    w, x, y, z = q
    return np.array([[1 - 2 * y ** 2 - 2 * z ** 2, 2 * x * y - 2 * w * z, 2 * z * x + 2 * w * y],
                     [2 * x * y + 2 * w * z, 1 - 2 * x ** 2 - 2 * z ** 2, 2 * y * z - 2 * w * x],
                     [2 * z * x - 2 * w * y, 2 * y * z + 2 * w * x, 1 - 2 * x ** 2 - 2 * y ** 2]])


def write_images(d, n, masks_d=None, zero_masks=False, size=(H, W)):
    os.makedirs(d, exist_ok=True)
    h, w = size
    yy, xx = np.mgrid[0:h, 0:w]
    for f in range(n):
        base = np.stack([np.sin(xx / (9.0 + 3 * c) + 0.4 * f) * np.cos(yy / (7.0 + 2 * c) - 0.2 * f) for c in range(3)], -1)
        Image.fromarray(np.clip(127.5 + 110 * base, 0, 255).astype(np.uint8)).save(os.path.join(d, '%05d.jpg' % f), quality=92)
        if masks_d is not None:
            os.makedirs(masks_d, exist_ok=True)
            m = np.zeros((h, w, 3), np.uint8)
            if not zero_masks:
                m[30 + 5 * f:90 + 5 * f, 120 + 10 * f:260 + 10 * f, 0] = 255
                m[5:20, 5:40, 1] = 255                                                # green only: not a motion mask
            Image.fromarray(m).save(os.path.join(masks_d, '%05d.png' % f))


def write_twin(root, sc, track='clip', zero_masks=False):
    """The scene as a DAVIS track under root (matrices.txt = inv(FLIP @ w2c), written with repr) and as COLMAP models
    root/sparse_bin and root/sparse_txt over the same image and mask files. -> (images_dir, masks_dir)"""
    n = sc['n']
    images_dir = os.path.join(root, 'JPEGImages', '1080p', track)
    masks_dir = os.path.join(root, 'Annotations', '1080p', track)
    write_images(images_dir, n, masks_dir, zero_masks)
    tri = os.path.join(root, 'triangulation')
    os.makedirs(tri, exist_ok=True)
    with open(os.path.join(tri, track + '.intrinsics.txt'), 'w') as f:
        f.writelines('%d %r %r %r %r\n' % (i, FX, FY, CX, CY) for i in range(n))
    with open(os.path.join(tri, track + '.matrices.txt'), 'w') as f:
        for i in range(n):
            f.write('%d ' % i + ' '.join(repr(float(v)) for v in np.linalg.inv(FLIP @ sc['w2c'][i]).reshape(-1)) + '\n')
    with open(os.path.join(tri, track + '.obj'), 'w') as f:
        f.writelines('v %r %r %r\n' % tuple(float(c) for c in p) for p in sc['xyz'])
    for form, writer in (('bin', write_bin), ('txt', write_txt)):
        writer(os.path.join(root, 'sparse_' + form), sc['cameras'], sc['images'], sc['points'])
    return images_dir, masks_dir


def bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.int64)


# ---- tests ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('exact', [True, False])
def test_text_and_binary_forms_read_bitwise_equal(tmp_path, exact):
    from dvd_b200 import frames as fr
    sc = scene(n=5, V=700, exact=exact, seed=3)
    write_bin(str(tmp_path / 'b'), sc['cameras'], sc['images'], sc['points'])
    write_txt(str(tmp_path / 't'), sc['cameras'], sc['images'], sc['points'])
    Kb, names_b, Eb, hb = fr.read_colmap_model(str(tmp_path / 'b'))
    Kt, names_t, Et, ht = fr.read_colmap_model(str(tmp_path / 't'))
    assert names_b == names_t == ['%05d.jpg' % f for f in range(5)]
    for a, b in ((Kb, Kt), (Eb, Et), (hb, ht)):
        assert a.dtype == b.dtype == np.float64 and a.shape == b.shape
        assert np.array_equal(bits(a), bits(b))
    # the values are the scene's: points ordered by id, cameras in the order of the names
    assert Eb.shape == (5, 4, 4) and hb.shape == (4, 700)
    assert np.array_equal(bits(hb[:3].T), bits(sc['xyz'])) and (hb[3] == 1).all()
    assert np.array_equal(bits(Eb), bits(sc['w2c']))
    # binary wins when both forms are present
    write_txt(str(tmp_path / 'b'), sc['cameras'][:2], sc['images'], sc['points'])         # the used camera missing
    assert np.array_equal(bits(fr.read_colmap_model(str(tmp_path / 'b'))[0]), bits(Kb))


def test_parameter_counts_skip_every_camera_model(tmp_path):
    """one camera of each model id before the used one: a wrong count anywhere misreads every later record"""
    from dvd_b200 import frames as fr
    sc = scene(n=2, V=50)
    g = np.random.default_rng(1)
    cams = [(100 + m, m, W, H, list(g.normal(size=k))) for m, (_, k) in MODELS.items()] + [sc['cameras'][-1]]
    write_bin(str(tmp_path / 'm'), cams, sc['images'], sc['points'])
    K = fr.read_colmap_model(str(tmp_path / 'm'))[0]
    assert np.array_equal(K, [[FX, 0, CX], [0, FY, CY], [0, 0, 1]])
    assert {m: k for m, (_, k) in fr.COLMAP_CAMERA_MODELS.items()} == {m: k for m, (_, k) in MODELS.items()}
    with open(str(tmp_path / 'm' / 'cameras.bin'), 'ab') as f:
        f.write(b'\0')
    with pytest.raises(ValueError, match='bytes after'):
        fr.read_colmap_model(str(tmp_path / 'm'))
    for part, cut in (('points3D', 9), ('images', 30), ('images', 3)):                # a file cut short, at any field
        write_bin(str(tmp_path / 'c'), sc['cameras'], sc['images'], sc['points'])
        path = str(tmp_path / 'c' / (part + '.bin'))
        with open(path, 'rb') as f:
            data = f.read()
        with open(path, 'wb') as f:
            f.write(data[:-cut])
        with pytest.raises(ValueError, match='ends inside'):
            fr.read_colmap_model(str(tmp_path / 'c'))
    # an unknown model id cannot be skipped
    write_bin(str(tmp_path / 'u'), [(1, 11, W, H, [1.0, 2.0])] + sc['cameras'], sc['images'], sc['points'])
    with pytest.raises(ValueError, match='unknown model id 11'):
        fr.read_colmap_model(str(tmp_path / 'u'))


def test_qvec2rotmat_matches_hand_built_rotations():
    from scipy.spatial.transform import Rotation
    from dvd_b200 import frames as fr
    s = np.sqrt(0.5)
    cases = [((1, 0, 0, 0), np.eye(3)),
             ((s, s, 0, 0), [[1, 0, 0], [0, 0, -1], [0, 1, 0]]),                  # 90 degrees about x
             ((s, 0, s, 0), [[0, 0, 1], [0, 1, 0], [-1, 0, 0]]),                  # about y
             ((s, 0, 0, s), [[0, -1, 0], [1, 0, 0], [0, 0, 1]]),                  # about z
             ((0.5, 0.5, 0.5, 0.5), [[0, 0, 1], [1, 0, 0], [0, 1, 0]])]           # 120 degrees about (1, 1, 1)
    for q, R in cases:
        got = fr.qvec2rotmat(q)
        assert got.dtype == np.float64 and got.shape == (3, 3)
        assert np.abs(got - np.asarray(R, np.float64)).max() <= 2 ** -52, q
        if 0.5 in q or q[0] == 1:
            assert np.array_equal(got, R), q                                      # exact where the products are
    g = np.random.default_rng(0)
    qs = g.normal(size=(50, 4))
    qs /= np.linalg.norm(qs, axis=1, keepdims=True)
    R = fr.qvec2rotmat(qs)
    assert R.shape == (50, 3, 3)
    assert np.abs(R - Rotation.from_quat(qs[:, [1, 2, 3, 0]]).as_matrix()).max() <= 1e-15
    assert all(np.array_equal(R[i], rotmat(qs[i])) for i in range(50))             # the batched form is the scalar one


@pytest.mark.parametrize('model', [0, 1])
def test_intrinsics_move_the_pixel_centre(tmp_path, model):
    from dvd_b200 import frames as fr
    sc = scene(n=2, V=20)
    params = [300.25, 211.0, 87.75] if model == 0 else [300.25, 310.5, 211.0, 87.75]
    write_txt(str(tmp_path), [(3, model, W, H, params)], sc['images'], sc['points'])
    K = fr.read_colmap_model(str(tmp_path))[0]
    fx, fy = (params[0], params[0]) if model == 0 else params[:2]
    assert np.array_equal(K, [[fx, 0, 211.0 - 0.5], [0, fy, 87.75 - 0.5], [0, 0, 1]])


def test_twin_readers_agree_bit_for_bit(tmp_path):
    from dvd_b200 import frames as fr
    sc = scene(n=6, V=2000)
    write_twin(str(tmp_path), sc)
    K, E, h_pt = fr.read_cameras(str(tmp_path), 'clip')
    for form in ('bin', 'txt'):
        Kc, names, Ec, hc = fr.read_colmap_model(str(tmp_path / ('sparse_' + form)))
        assert names == sorted(os.listdir(str(tmp_path / 'JPEGImages' / '1080p' / 'clip')))
        for a, b in ((Kc, K), (Ec, E), (hc, h_pt)):
            assert a.shape == b.shape and np.array_equal(bits(a), bits(b))


def test_twin_readers_agree_within_ulps_for_general_rotations(tmp_path):
    from dvd_b200 import frames as fr
    sc = scene(n=6, V=500, exact=False, seed=5)
    write_twin(str(tmp_path), sc)
    K, E, h_pt = fr.read_cameras(str(tmp_path), 'clip')
    Kc, _, Ec, hc = fr.read_colmap_model(str(tmp_path / 'sparse_bin'))
    assert np.array_equal(bits(Kc), bits(K)) and np.array_equal(bits(hc), bits(h_pt))
    # the DAVIS file holds the inverse of the flipped matrix: two inversions in fp64
    assert np.abs(Ec - E).max() <= 8 * 2 ** -52 * np.abs(E).max()


def write_model(d, sc, cameras=None, images=None, points=None):
    write_bin(d, sc['cameras'] if cameras is None else cameras, sc['images'] if images is None else images,
              sc['points'] if points is None else points)
    return d


def test_rejections(tmp_path):
    from dvd_b200 import frames as fr
    sc = scene(n=3, V=100)
    images_dir = str(tmp_path / 'images')
    write_images(images_dir, 3)
    ok = write_model(str(tmp_path / 'ok'), sc)

    def build(model_dir, images=images_dir, masks=None):
        # every check runs before the network is touched
        return fr.ColmapFrameBuilder(images, model_dir, None, masks_dir=masks)

    radial = [c if c[0] != 3 else (3, 2, W, H, [FX, CX, CY, 0.01]) for c in sc['cameras']]
    with pytest.raises(ValueError, match='colmap image_undistorter'):
        build(write_model(str(tmp_path / 'radial'), sc, cameras=radial))
    two = [im if im[4] != '00001.jpg' else im[:3] + (5,) + im[4:] for im in sc['images']]
    with pytest.raises(ValueError, match='2 cameras'):
        build(write_model(str(tmp_path / 'two'), sc, cameras=sc['cameras'] + [(5, 1, W, H, [FX, FY, CX, CY])], images=two))
    with pytest.raises(ValueError, match='no 3-D point'):
        build(write_model(str(tmp_path / 'nopts'), sc, points=[]))
    with pytest.raises(ValueError, match='no registered image'):
        build(write_model(str(tmp_path / 'noimg'), sc, images=[]))
    small = [c if c[0] != 3 else (3, 1, W, H - 32, c[4]) for c in sc['cameras']]
    with pytest.raises(ValueError, match='00000.jpg is 160x416'):
        build(write_model(str(tmp_path / 'size'), sc, cameras=small))
    # an image file the model did not register, in any case of the extension and in a subdirectory
    for extra in ('00003.JPG', 'more/x.png'):
        path = os.path.join(images_dir, extra)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        Image.new('RGB', (W, H)).save(path, format='PNG')
        with pytest.raises(ValueError, match='not registered.*%s' % extra.replace('.', r'\.')):
            build(ok)
        os.remove(path)
    with open(os.path.join(images_dir, 'notes.txt'), 'w') as f:
        f.write('not an image')
    with pytest.raises(FileNotFoundError, match='mask'):
        build(ok, masks=str(tmp_path / 'no_masks'))                                # other files are ignored; masks checked
    os.remove(os.path.join(images_dir, '00002.jpg'))
    with pytest.raises(FileNotFoundError, match='00002.jpg'):
        build(ok)
    with pytest.raises(FileNotFoundError):
        fr.read_colmap_model(str(tmp_path / 'images'))
    with pytest.raises(ValueError, match='chunk'):
        fr.ColmapFrameBuilder(images_dir, ok, None, chunk=0)


def test_cli_source_arguments(tmp_path):
    from dvd_b200 import prepare_frames
    base = ['--midas_ckpt', 'x.pt', '--out', str(tmp_path)]
    for argv in (['--colmap_model', 'm'], ['--davis_root', 'd', '--track', 't', '--images', 'i'],
                 ['--colmap_model', 'm', '--davis_root', 'd', '--images', 'i'], ['--colmap_model', 'm', '--images', 'i', '--track', 't']):
        with pytest.raises(SystemExit):
            prepare_frames.main(argv + base)
