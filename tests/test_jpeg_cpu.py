"""Device JPEG decoding without a GPU: the header parser's device / host decisions, and csrc/pf_jpeg.cu compiled for
the host (-DPF_JPEG_HOST_TEST) against Pillow bit for bit, on a seeded fixture matrix; the --enbl_device_decode input
pipeline end to end with that host build standing in for the kernels."""
import os
import shutil

import numpy as np
import pytest

pytest.importorskip('PIL.Image')
import jpeg_fixtures as F  # noqa: E402
from pocketflow_b200.datasets import jpeg as J  # noqa: E402
from jpeg_fixtures import decode_jpeg, jpeg_shape  # noqa: E402,F401

needs_gxx = pytest.mark.skipif(shutil.which('g++') is None, reason='no host compiler')


@pytest.fixture(scope='module')
def host_lib(tmp_path_factory):
    if shutil.which('g++') is None:
        pytest.skip('no host compiler')
    return F.host_decoder(tmp_path_factory.mktemp('jpeg_host'))


def run_host(lib, items):
    descs, scans, ws, nbytes, layout = F.batch(items)
    out = np.zeros(max(nbytes, 1), np.uint8)
    wsb = np.zeros(max(ws, 64), np.int16)
    status = np.full(len(items), -1, np.int32)
    lib.pf_test_jpeg_decode_host(scans.ctypes.data, descs.ctypes.data, len(items), wsb.ctypes.data, out.ctypes.data,
                                 status.ctypes.data)
    return status, [out[o:o + int(np.prod(s))].reshape(s) for o, s in layout]


def test_descriptor_layout_matches_the_c_struct(host_lib):
    assert host_lib.pf_test_jpeg_desc_size() == J.JPEG_DESC.itemsize == 4144
    assert J.JPEG_DESC.fields['quant'][1] == 112 and J.JPEG_DESC.fields['huff'][1] == 496


def test_parser_decisions_and_shapes():
    for name, buf in F.device_matrix():
        h = J.parse_header(buf)
        assert h.device, (name, h.reason)
        assert (h.height, h.width) == jpeg_shape(buf), name
        assert buf[h.scan_start + h.scan_bytes - 2:h.scan_start + h.scan_bytes] == b'\xff\xd9'
    want = {'progressive': 'SOF2', 'progressive_L': 'SOF2', 'cmyk': '4 components', 'png': 'not a JPEG',
            'truncated': 'EOI', 'empty': 'not a JPEG'}
    for name, buf in F.host_matrix():
        h = J.parse_header(buf)
        assert not h.device and want[name] in h.reason, (name, h.reason)
        if name not in ('png', 'empty'):
            assert (h.height, h.width) == jpeg_shape(buf), name


def test_parser_restates_libjpeg_colour_space_rules():
    """default_decompress_parms: JFIF means YCbCr; without it an Adobe transform decides, and without either the
    component ids ('R', 'G', 'B' means RGB)."""
    buf = F.jpeg(16, 16, 1, '444')
    assert buf[2:4] == b'\xff\xe0' and J.parse_header(buf).device
    seg = 2 + int.from_bytes(buf[4:6], 'big')
    bare = buf[:2] + buf[2 + seg:]                                    # no JFIF marker, component ids 1, 2, 3
    assert J.parse_header(bare).device and np.array_equal(decode_jpeg(bare), decode_jpeg(buf))
    sof = bare.index(b'\xff\xc0')
    rgb = bytearray(bare)
    for i, cid in enumerate(b'RGB'):
        rgb[sof + 10 + 3 * i] = cid
    sos = rgb.index(b'\xff\xda')
    for i, cid in enumerate(b'RGB'):
        rgb[sos + 5 + 2 * i] = cid
    assert J.parse_header(bytes(rgb)).reason == 'RGB colour space'
    for transform, device in ((0, False), (1, True)):
        adobe = b'\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00' + bytes([transform])
        assert J.parse_header(bare[:2] + adobe + bare[2:]).device == device
    for sub, ok in (('444', True), ('422', True), ('420', True)):
        assert J.parse_header(F.jpeg(24, 40, 2, sub)).device == ok
    b440 = bytearray(F.jpeg(24, 40, 3, '444'))
    sof = b440.index(b'\xff\xc0')
    b440[sof + 11] = 0x12                                             # luma 1x2: 4:4:0
    assert 'sampling' in J.parse_header(bytes(b440)).reason


@needs_gxx
def test_host_compiled_kernels_equal_pillow_bit_for_bit(host_lib):
    """Every device fixture, with the whole image, an interior window and windows touching each edge, all decoded in
    one call (one descriptor per window, workspaces and crops back to back)."""
    checked = 0
    for name, buf in F.device_matrix():
        h = J.parse_header(buf)
        windows = F.crops(h.height, h.width)
        status, got = run_host(host_lib, [(buf, c) for c in windows])
        assert (status == 0).all(), (name, status)
        for c, g in zip(windows, got):
            np.testing.assert_array_equal(g, decode_jpeg(buf, c), err_msg='%s crop %s' % (name, c))
            checked += 1
    assert checked > 600


@needs_gxx
def test_anomalies_flag_only_their_own_image(host_lib):
    good = [F.jpeg(64, 48, 1, '420'), F.jpeg(40, 72, 2, 'L', restart_marker_rows=1), F.jpeg(33, 17, 3, '422', 100)]
    bad_code = F.corrupt_huffman(F.jpeg(128, 96, 4, '420', restart_marker_blocks=5))
    bad_code_plain = F.corrupt_huffman(F.jpeg(200, 150, 5, '444'))
    items = [(good[0], None), (bad_code, None), (good[1], None), (bad_code_plain, None), (good[2], (3, 2, 20, 11))]
    status, got = run_host(host_lib, items)
    assert status[1] in (1, 4) and status[3] in (1, 4), status
    assert (status[[0, 2, 4]] == 0).all()
    for i in (0, 2, 4):
        np.testing.assert_array_equal(got[i], decode_jpeg(items[i][0], items[i][1]))
    # a scan cut short: the kernel runs out of data and says so, the neighbours are untouched
    descs, scans, ws, nbytes, layout = F.batch([(good[0], None), (F.jpeg(120, 160, 6, '420'), None), (good[2], None)])
    descs['scan_bytes'][1] //= 3
    out, wsb, st = np.zeros(nbytes, np.uint8), np.zeros(ws, np.int16), np.full(3, -1, np.int32)
    host_lib.pf_test_jpeg_decode_host(scans.ctypes.data, descs.ctypes.data, 3, wsb.ctypes.data, out.ctypes.data,
                                      st.ctypes.data)
    assert st.tolist() == [0, 2, 0]
    for i in (0, 2):
        o, s = layout[i]
        np.testing.assert_array_equal(out[o:o + int(np.prod(s))].reshape(s), decode_jpeg([good[0], None, good[2]][i]))


@needs_gxx
def test_descriptors_outside_the_decoded_window_are_refused(host_lib):
    """A descriptor that would send the kernels past the image, or past the MCU window whose blocks were decoded and
    transformed, sets status 5 and leaves the other images alone.  64x48 4:2:0, rows 8..47: luma reads MCU rows 0..2,
    the upsampler's chroma context row 24 reads MCU row 3; columns 0..47 read MCU columns 0..2."""
    img, other = F.jpeg(64, 48, 1, '420'), F.jpeg(40, 72, 2, 'L')
    descs, scans, ws, nbytes, layout = F.batch([(img, (8, 0, 40, 48)), (other, None)])
    assert descs['mcu_rows'][0] == 4 and descs['mcu_row0'][0] == 0 and descs['mcu_col1'][0] == 2
    for field, value in (('crop_h', 10 ** 6), ('mcu_rows', 3), ('mcu_row0', 1), ('mcu_col1', 1)):
        bad = descs.copy()
        bad[field][0] = value
        out, wsb, st = np.zeros(nbytes, np.uint8), np.zeros(ws, np.int16), np.full(2, -1, np.int32)
        host_lib.pf_test_jpeg_decode_host(scans.ctypes.data, bad.ctypes.data, 2, wsb.ctypes.data, out.ctypes.data,
                                          st.ctypes.data)
        assert st.tolist() == [5, 0], (field, st)
        o, shape = layout[1]
        np.testing.assert_array_equal(out[o:o + int(np.prod(shape))].reshape(shape), decode_jpeg(other))
    status, got = run_host(host_lib, [(img, (8, 0, 40, 48))])
    assert status[0] == 0
    np.testing.assert_array_equal(got[0], decode_jpeg(img, (8, 0, 40, 48)))


@needs_gxx
def test_device_decode_pipeline_equals_the_host_pipeline(tmp_path, monkeypatch, host_lib):
    """--enbl_device_decode end to end on the CPU: the parser and crop draws in the worker pool, DecodeBatchIterator,
    AbstractLearner._feed_decoded with pf_jpeg_decode and pf_preprocess_images replaced by their host builds; the
    placeholders get exactly the host pipeline's batches, training and evaluation, over shards with progressive, CMYK,
    PNG and corrupted files."""
    import torch
    from pocketflow_b200 import ops
    pre = F.host_preprocessor(tmp_path)
    calls = {'decoded': 0, 'flagged': 0}

    def preprocess_on_host(crops, desc, out, mean=(123.68, 116.78, 103.94)):
        pre(crops.data_ptr(), desc.data_ptr(), out.shape[0], out.shape[1], out.shape[2], mean[0], mean[1], mean[2],
            out.data_ptr())
        return out

    def decode_on_host(data, desc, n, ws, crops, status):
        assert data.dtype == torch.uint8 and ws.dtype == torch.int16 and status.dtype == torch.int32
        host_lib.pf_test_jpeg_decode_host(data.data_ptr(), desc.data_ptr(), n, ws.data_ptr(), crops.data_ptr(),
                                          status.data_ptr())
        calls['decoded'] += n
        calls['flagged'] += int((status[:n] != 0).sum())
        return status
    monkeypatch.setattr(ops, 'preprocess_images', preprocess_on_host)
    monkeypatch.setattr(ops, 'jpeg_decode', decode_on_host)
    d = str(tmp_path / 'data')
    F.write_shards(d)
    for is_train in (True, False):
        host, _ = F.pipeline_batches(d, 'host', is_train, 6)
        dev, _ = F.pipeline_batches(d, 'decode', is_train, 6)
        for k, ((hi, hl), (di, dl)) in enumerate(zip(host, dev)):
            np.testing.assert_array_equal(dl, hl)
            np.testing.assert_array_equal(di, hi, err_msg='batch %d, training %s' % (k, is_train))
    assert calls['decoded'] > 20 and calls['flagged'] > 0


def test_truncated_files_raise_what_the_host_pipeline_raises(tmp_path):
    """A file cut short goes to the host decoder, so the pipeline fails the way the host pipeline does."""
    d = str(tmp_path / 'data')
    os.makedirs(d)
    F.R.write_records(os.path.join(d, "train-00000-of-00001"),
                    [F.example(F.jpeg(120, 160, 5)[:-700], 3)] + [F.example(F.jpeg(100, 100, i), 4) for i in range(3)])
    with pytest.raises(OSError):
        decode_jpeg(F.jpeg(120, 160, 5)[:-700])
    for mode in ('host', 'decode'):
        with pytest.raises(RuntimeError) as err:
            F.pipeline_batches(d, mode, True, 2, b=4)
        assert isinstance(err.value.__cause__, OSError)
