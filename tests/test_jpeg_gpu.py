"""pf_jpeg_decode on the GPU against Pillow, bit for bit: the fixture matrix at batch 1, at an odd batch and as 256
mixed images in one launch; a corrupted image flags only itself; the --enbl_device_decode feed equals the host
pipeline over TFRecord shards that hold fallback files."""
import numpy as np
import pytest
import torch

pytest.importorskip('PIL.Image')
import jpeg_fixtures as F  # noqa: E402
from pocketflow_b200 import ops  # noqa: E402
from jpeg_fixtures import decode_jpeg, jpeg_shape  # noqa: E402,F401

pytestmark = pytest.mark.gpu


def run_device(items):
    descs, scans, ws, nbytes, layout = F.batch(items)
    dev = torch.device('cuda')
    data = torch.from_numpy(np.concatenate([scans, np.zeros(1, np.uint8)])).to(dev)
    desc = torch.from_numpy(descs.view(np.uint8).reshape(-1).copy()).to(dev)
    ws_t = torch.full((max(ws, 64),), 0x7BCD, dtype=torch.int16, device=dev)
    crops = torch.full((max(nbytes, 1),), 0xA5, dtype=torch.uint8, device=dev)
    status = torch.full((len(items),), -1, dtype=torch.int32, device=dev)
    ops.jpeg_decode(data, desc, len(items), ws_t, crops, status)
    torch.cuda.synchronize()
    out = crops.cpu().numpy()
    return status.cpu().numpy(), [out[o:o + int(np.prod(s))].reshape(s) for o, s in layout]


def check(items, status, got):
    for (buf, crop), s, g in zip(items, status, got):
        assert s == 0
        np.testing.assert_array_equal(g, decode_jpeg(buf, crop))


def test_matrix_at_batch_1_and_at_odd_batches():
    """Every fixture alone, whole image; then every fixture with every crop window, seven fixtures per launch, made
    odd by one more whole image where the count is even."""
    matrix = F.device_matrix()
    for name, buf in matrix:
        items = [(buf, None)]
        check(items, *run_device(items))
    for k in range(0, len(matrix), 7):
        items = []
        for name, buf in matrix[k:k + 7]:
            h = F.J.parse_header(buf)
            items += [(buf, c) for c in F.crops(h.height, h.width)]
        if len(items) % 2 == 0:
            items.append((matrix[k][1], None))
        check(items, *run_device(items))


def test_256_mixed_images_in_one_launch():
    matrix = F.device_matrix()
    rng = np.random.RandomState(0)
    items = []
    for i in range(256):
        name, buf = matrix[i % len(matrix)]
        h = F.J.parse_header(buf)
        c = F.crops(h.height, h.width)
        items.append((buf, c[rng.randint(len(c))]))
    check(items, *run_device(items))


def test_a_corrupted_image_flags_only_itself():
    good = [F.jpeg(500, 375, 1, '420'), F.jpeg(255, 257, 2, 'L', restart_marker_rows=1), F.jpeg(33, 17, 3, '422', 100)]
    bad = F.corrupt_huffman(F.jpeg(375, 500, 4, '420', restart_marker_blocks=5))
    items = [(good[0], None), (bad, None), (good[1], (5, 7, 100, 200)), (good[2], None)]
    status, got = run_device(items)
    assert status[1] in (1, 4) and (status[[0, 2, 3]] == 0).all(), status
    for i in (0, 2, 3):
        np.testing.assert_array_equal(got[i], decode_jpeg(*items[i]))


def test_device_decode_feed_equals_the_host_pipeline(tmp_path):
    d = str(tmp_path / 'data')
    F.write_shards(d)
    for is_train in (True, False):
        host, _ = F.pipeline_batches(d, 'host', is_train, 6)
        dev, _ = F.pipeline_batches(d, 'decode', is_train, 6)
        for (hi, hl), (di, dl) in zip(host, dev):
            np.testing.assert_array_equal(dl, hl)
            np.testing.assert_array_equal(di, hi)
