"""CPU: dataset_tool against the reference's own dataset_tool.py (tests/golden/make_dataset_tool_golden.py), and the resampler's
restatement (oracle/resample.py) against PIL.

  - oracle.resample (numpy int64: Pillow's tables, both passes, skipped passes and the ybox) equals PIL.Image.resize(LANCZOS) byte for
    byte, and the product's tables (torch_utils/ops/resample.lanczos_tables) are the oracle's;
  - the port's command, with ide3d_resample_u8 swapped for the oracle and the device for the CPU, reproduces every golden case: archive
    names, pixels, dataset.json text, stdout, exit codes and exceptions.  JPEG pixels are compared with the golden under the Pillow
    version that wrote it, and otherwise with PIL's JPEG coding, run live, of the paired PNG case's pixels;
  - --seg-dest: with a seeded BiSeNet and the labels kernel swapped for its oracle, every mask is the face_parsing composition, and
    train_encoder.PortraitDataset reads the pairs with their flipped camera labels.
"""

import io
import json
import os
import sys
import zipfile

import numpy as np
import PIL
import PIL.Image
import pytest
import torch
import torch.nn.functional as F
from click.testing import CliRunner

from conftest import ROOT, load_golden

sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
import make_dataset_tool_golden as dg  # noqa: E402

from ide3d_b200 import dataset_tool, parsing  # noqa: E402
from ide3d_b200.torch_utils.ops import resample as ops  # noqa: E402
from ide3d_b200.torch_utils.ops import seg_stem as seg_ops  # noqa: E402
from oracle import finetune as ofin  # noqa: E402
from oracle import resample as ores  # noqa: E402

SIZES = [((1024, 1024), (512, 512)), ((1024, 1024), (256, 256)), ((1000, 1000), (512, 512)), ((512, 512), (512, 512)),
         ((256, 256), (512, 512)), ((7, 3), (2, 5)), ((300, 200), (128, 96)), ((200, 300), (64, 64)), ((300, 200), (300, 100)),
         ((300, 200), (150, 200))]                                                # (w, h) -> (w, h); the last two skip one pass


def test_image(w, h, channels, kind, seed=0):
    rng = np.random.default_rng(seed)
    shape = (h, w) if channels == 1 else (h, w, channels)
    if kind == 'noise':
        return rng.integers(0, 256, shape, dtype=np.uint8)
    yy, xx = np.mgrid[0:h, 0:w]
    a = ((np.sin(xx / 17.0) + np.cos(yy / 23.0)) * 60 + 128).astype(np.uint8)
    return a if channels == 1 else np.stack([a, 255 - a, a // 2], -1)


test_image.__test__ = False


@pytest.mark.parametrize('src, dst', SIZES, ids=[f'{a[0]}x{a[1]}-{b[0]}x{b[1]}' for a, b in SIZES])
@pytest.mark.parametrize('channels', [1, 3])
@pytest.mark.parametrize('kind', ['noise', 'smooth'])
def test_oracle_equals_pil(src, dst, channels, kind):
    img = test_image(*src, channels, kind)
    want = np.array(PIL.Image.fromarray(img).resize(dst, PIL.Image.LANCZOS))
    got = ores.resize(img, dst)
    assert got.dtype == np.uint8 and got.shape == want.shape and np.array_equal(got, want)


@pytest.mark.parametrize('n_in, n_out', [(1024, 512), (1024, 256), (1000, 512), (512, 512), (256, 512), (7, 2), (3, 5), (70, 3)])
def test_product_tables_are_pillows(n_in, n_out):
    k1, b1, c1 = ops.lanczos_tables(n_in, n_out)
    k2, b2, c2 = ores.lanczos_tables(n_in, n_out)
    assert k1 == k2 and np.array_equal(b1, b2) and np.array_equal(c1, c2)


# ------------------------------------------------------------------------------------------------------------------------ the command
def oracle_resample_u8(src, dst):
    """ide3d_resample_u8 on CPU tensors through oracle.resample, image by image."""
    for i in range(src.shape[0]):
        a = src[i].numpy()
        r = ores.resize(a[:, :, 0] if a.shape[2] == 1 else a, (dst.shape[2], dst.shape[1]))
        dst[i].copy_(torch.from_numpy(r.reshape(dst.shape[1:])))
    return dst


@pytest.fixture
def cpu_tool(monkeypatch):
    monkeypatch.setattr(ops, 'resample_u8', oracle_resample_u8)
    monkeypatch.setattr(dataset_tool, '_device', lambda: torch.device('cpu'))


@pytest.fixture(scope='module')
def golden():
    return load_golden('dataset_tool')


@pytest.fixture(scope='module')
def sources(tmp_path_factory):
    root = str(tmp_path_factory.mktemp('dataset_tool_src'))
    dg.make_sources(root)
    return root


def jpeg_roundtrip(px):
    b = io.BytesIO()
    PIL.Image.fromarray(px).save(b, format='jpeg', quality=100)
    return np.array(PIL.Image.open(b))


def check_case(golden, name, rec, root):
    g = lambda k: golden[f'{name}/{k}']
    assert rec['exit_code'] == int(g('exit_code'))
    assert rec['stdout'].replace(root, '<src>') == str(g('stdout'))
    assert rec['exception'] == str(g('exception'))
    assert rec['json'] == str(g('json'))
    assert sorted(rec['images']) == list(g('names'))
    live = name in dg.JPEG_OF and str(golden['pillow_version']) != PIL.__version__
    for n, px in rec['images'].items():
        want = jpeg_roundtrip(golden[f'{dg.JPEG_OF[name]}/px/{n}']) if live else golden[f'{name}/px/{n}']
        assert px.dtype == want.dtype and px.shape == want.shape and np.array_equal(px, want), n


@pytest.mark.parametrize('name', sorted(dg.CASES))
def test_command_reproduces_reference(golden, sources, tmp_path, cpu_tool, name):
    workers = ['--workers', '2'] if name.startswith(('folder', 'zip')) else ['--workers', '0']
    rec = dg.run_case(dataset_tool.convert_dataset, sources, str(tmp_path), name, workers)
    check_case(golden, name, rec, sources)


@pytest.mark.parametrize('name', ['folder_scale_zip', 'zip_crop_wide'])
def test_batch_size_does_not_change_output(golden, sources, tmp_path, cpu_tool, monkeypatch, name):
    monkeypatch.setattr(dataset_tool, 'DEFAULT_BATCH', 2)
    rec = dg.run_case(dataset_tool.convert_dataset, sources, str(tmp_path), name, ['--workers', '1'])
    check_case(golden, name, rec, sources)


@pytest.mark.parametrize('source, message', [('x_lmdb', 'LSUN LMDB sources are not supported'),
                                             ('cifar-10-python.tar.gz', 'CIFAR-10 and MNIST sources are not supported'),
                                             ('train-images-idx3-ubyte.gz', 'CIFAR-10 and MNIST sources are not supported'),
                                             ('missing', 'Missing input file or directory')])
def test_refused_sources(tmp_path, cpu_tool, source, message):
    path = tmp_path / source
    if source.endswith('_lmdb'):
        path.mkdir()
    elif source != 'missing':
        path.write_bytes(b'')
    r = CliRunner(mix_stderr=False).invoke(dataset_tool.convert_dataset, ['--source', str(path), '--dest', str(tmp_path / 'o.zip')])
    assert r.exit_code == 1 and r.stdout.startswith('Error: ') and message in r.stdout


def test_seg_dest_needs_parser(tmp_path, cpu_tool, sources):
    r = CliRunner(mix_stderr=False).invoke(dataset_tool.convert_dataset, ['--source', os.path.join(sources, 'folder_plain'), '--dest',
                                                                          str(tmp_path / 'o.zip'), '--seg-dest', str(tmp_path / 's')])
    assert r.exit_code == 2 and '--seg-dest and --parser must be given together' in r.stderr


def test_device_is_required(tmp_path, sources, monkeypatch):
    monkeypatch.setattr(torch.cuda, 'is_available', lambda: False)
    r = CliRunner(mix_stderr=False).invoke(dataset_tool.convert_dataset, ['--source', os.path.join(sources, 'folder_plain'), '--dest',
                                                                          str(tmp_path / 'o.zip'), '--workers', '0'])
    assert r.exit_code == 1 and 'needs a CUDA device' in r.stdout


# ----------------------------------------------------------------------------------------------------------------------------- masks
CAMERA = np.array([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 2.7, 0, 0, 0, 1, 4.2647, 0, 0.5, 0, 4.2647, 0.5, 0, 0, 1], dtype=np.float64)


def portrait_source(root, n=3, size=64, seed=3):
    rng = np.random.default_rng(seed)
    labels = []
    for i in range(n):
        img = dg._smooth(rng, size + 8 * i, size, 3)
        PIL.Image.fromarray(img).save(os.path.join(root, f'p{i}.png'))
        labels.append([f'p{i}.png', (CAMERA + 0.01 * i).tolist()])
    with open(os.path.join(root, 'dataset.json'), 'w') as f:
        json.dump({'labels': labels}, f)


def face_parsing(net, img):
    """dnnlib/seg_tools.face_parsing(x / 127.5 - 1) as the reference composes it: resize to 512^2 (align_corners=True), BiSeNet,
    the upsampled logits' argmax (the oracle of ide3d_seg_labels_ac) and id_remap."""
    x = torch.from_numpy(img).permute(2, 0, 1)[None].float() / 127.5 - 1
    x = F.interpolate(x, size=(512, 512), mode='bilinear', align_corners=True)
    return parsing.remap_ids(ofin.seg_labels(net.logits(x), (512, 512), align_corners=True))[0].numpy()


@pytest.mark.parametrize('dest_kind', ['zip', 'dir'])
def test_seg_dest_masks_and_portrait_dataset(tmp_path, cpu_tool, monkeypatch, dest_kind):
    monkeypatch.setattr(seg_ops, 'seg_labels', ofin.seg_labels)
    src = tmp_path / 'src'
    src.mkdir()
    portrait_source(str(src))
    net = parsing.BiSeNet()
    net.load_state_dict(ofin.bisenet_state(net))
    torch.save(net.state_dict(), tmp_path / 'bisenet.pth')
    net.eval()
    sfx = '.zip' if dest_kind == 'zip' else ''
    dest, seg = str(tmp_path / ('out' + sfx)), str(tmp_path / ('seg' + sfx))
    r = CliRunner(mix_stderr=False).invoke(dataset_tool.convert_dataset, [
        '--source', str(src), '--dest', dest, '--transform', 'center-crop', '--resolution', '64x64', '--seg-dest', seg,
        '--parser', str(tmp_path / 'bisenet.pth'), '--workers', '2'])
    assert r.exit_code == 0, (r.stdout, r.exception)
    images, _ = dg.read_dest(dest)
    masks, seg_json = dg.read_dest(seg)
    assert sorted(masks) == sorted(images) and len(images) == 3 and seg_json == ''
    with torch.no_grad():
        for n, img in images.items():
            assert masks[n].dtype == np.uint8 and masks[n].shape == (512, 512)
            assert np.array_equal(masks[n], face_parsing(net, img)), n

    from ide3d_b200 import train_encoder
    ds = train_encoder.PortraitDataset(dest, seg, 64)
    assert len(ds) == 3
    for i in range(3):
        image, mask, label = ds[i]
        name = f'00000/img{i:08d}.png'
        assert np.array_equal(image.permute(1, 2, 0).numpy(), images[name])
        assert np.array_equal(mask.numpy(), np.array(PIL.Image.fromarray(masks[name]).resize((64, 64), PIL.Image.NEAREST)))
        want = CAMERA + 0.01 * i
        want[train_encoder.LABEL_FLIP] *= -1
        assert np.allclose(label.numpy(), want.astype(np.float32))


def test_product_resample_refuses_cpu_and_bad_operands():
    with pytest.raises(RuntimeError, match='CUDA device'):
        ops.resize_u8(torch.zeros(1, 8, 8, 3, dtype=torch.uint8), (4, 4))


def test_abi_refuses_bad_arguments(lib):
    from ide3d_b200 import _lib
    kx, bx, cx = ops.lanczos_tables(8, 4)
    ptr = lambda a: a.ctypes.data
    fake = 0x10000
    good = dict(inp=fake, n=1, c=3, in_h=8, in_w=8, out=fake, out_h=4, out_w=4, kx=kx, bx=ptr(bx), cx=ptr(cx), ky=kx, by=ptr(bx),
                cy=ptr(cx), scratch=fake, bytes=1 << 20)

    def call(**kw):
        a = dict(good, **kw)
        return lib.ide3d_resample_u8(a['inp'], a['n'], a['c'], a['in_h'], a['in_w'], 8 * 8 * 3, 8 * 3, 3, a['out'], a['out_h'],
                                     a['out_w'], 48, 12, 3, a['kx'], a['bx'], a['cx'], a['ky'], a['by'], a['cy'], a['scratch'],
                                     a['bytes'], None)

    bad_bounds = bx.copy()
    bad_bounds[2] = 7, 4
    for kw, msg in [(dict(inp=None), b'null input'), (dict(bx=None), b'null table'), (dict(c=4), b'4 channels'),
                    (dict(c=2), b'2 channels'), (dict(n=0), b'bad sizes'), (dict(in_w=-1), b'bad sizes'), (dict(kx=0), b'bad ksize'),
                    (dict(in_w=5), b'horizontal table entry'), (dict(in_h=6), b'vertical table entry'),
                    (dict(bx=ptr(bad_bounds)), b'horizontal table entry'), (dict(kx=2), b'horizontal table entry'),
                    (dict(scratch=None), b'null scratch'), (dict(scratch=fake + 4), b'16-byte aligned'), (dict(bytes=16), b'scratch of')]:
        assert call(**kw) == _lib.INVALID, kw
        assert msg in lib.ide3d_last_error(), (kw, lib.ide3d_last_error())
    assert lib.ide3d_resample_u8_scratch_bytes(1, 2, 8, 4, 4, 13, 13) == _lib.INVALID
    assert lib.ide3d_resample_u8_scratch_bytes(1, 3, 8, 4, 4, 13, 13) > 4 * 8 * 3
