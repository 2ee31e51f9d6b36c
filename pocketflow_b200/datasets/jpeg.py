"""JPEG header parser for device decoding (pf_jpeg_decode, csrc/pf_jpeg.cu).

`parse_header(buf)` walks the markers of one file and decides whether the device can decode it bit for bit with
libjpeg-turbo as Pillow runs it (`ilsvrc12_dataset.decode_jpeg`).  The device takes only baseline files: 8-bit
samples, one interleaved sequential Huffman scan (SOF0 / SOF1) followed by EOI, one component or three components that
libjpeg treats as YCbCr, luma sampling 1x1, 2x1 or 2x2 and chroma 1x1.  Everything else — progressive or arithmetic
coding, 12-bit samples, CMYK / YCCK / RGB, 4:4:0 and 4:1:1, several scans, a missing EOI, tables libjpeg would reject,
bytes that are not a JPEG — is decoded by the host.  `descriptor(...)` turns a parsed header and a crop window into
the fixed-size pf_jpeg_desc record the kernels read."""
import functools

import numpy as np

HUFF = np.dtype([('lookup', '<i2', 256), ('maxcode', '<i4', 18), ('valoffset', '<i4', 18), ('huffval', 'u1', 256)])
JPEG_DESC = np.dtype([
    ('scan_offset', '<i8'), ('coef_offset', '<i8'), ('crop_offset', '<i8'), ('scan_bytes', '<i4'),
    ('height', '<i4'), ('width', '<i4'), ('ncomp', '<i4'), ('hs', '<i4'), ('vs', '<i4'), ('restart_interval', '<i4'),
    ('mcus_per_row', '<i4'), ('mcu_rows', '<i4'), ('mcu_row0', '<i4'), ('mcu_col0', '<i4'), ('mcu_col1', '<i4'),
    ('crop_y', '<i4'), ('crop_x', '<i4'), ('crop_h', '<i4'), ('crop_w', '<i4'), ('dc_tbl', '<i4', 3),
    ('ac_tbl', '<i4', 3), ('quant', '<u2', (3, 64)), ('huff', HUFF, 4)])          # pf_jpeg_desc (include/pf_b200.h)
assert JPEG_DESC.itemsize == 4144

STATUS = {0: 'ok', 1: 'bad Huffman code', 2: 'data ends early', 3: 'bad restart marker', 4: 'run past coefficient 63',
          5: 'bad descriptor'}



def scan_end(buf, start):
    """Offset just past the marker that ends the entropy-coded segment starting at `start` — the first 0xFF followed by
    anything but a stuffed zero, RSTn or more fill — and that marker's code; (len(buf), None) if there is none.
    Vectorised: a Python loop or regex over every scan byte would cost as much as decoding the file."""
    a = np.frombuffer(buf, np.uint8, offset=start)
    ff = np.flatnonzero(a[:-1] == 0xFF)
    nxt = a[ff + 1]
    end = ff[(nxt != 0) & (nxt != 0xFF) & ((nxt < 0xD0) | (nxt > 0xD7))]
    if not len(end):
        return len(buf), None
    return start + int(end[0]) + 2, int(a[end[0] + 1])


class Header(object):
    """What the parser learned.  `device` says whether pf_jpeg_decode may decode the file; `reason` why not."""

    def __init__(self):
        self.device, self.reason = False, ''
        self.height = self.width = 0
        self.ncomp, self.hs, self.vs, self.restart_interval = 0, 1, 1, 0
        self.scan_start = self.scan_bytes = 0
        self.quant = None            # [ncomp, 64] uint16, zig-zag order
        self.tables = []             # derived Huffman tables (HUFF records), at most 4
        self.dc_tbl, self.ac_tbl = [0, 0, 0], [0, 0, 0]

    def host(self, reason):
        self.device, self.reason = False, reason
        return self


@functools.lru_cache(maxsize=256)
def derive_huffman(bits, vals, is_dc):
    """jdhuff.c jpeg_make_d_derived_tbl: one HUFF record, or None where libjpeg would reject the table.  bits / vals
    are the DHT segment's bytes; most files carry the same few tables, so the result is cached (callers copy it)."""
    t = np.zeros((), HUFF)
    huffsize = [l for l in range(1, 17) for _ in range(bits[l - 1])]
    if len(huffsize) > 256 or len(vals) < len(huffsize):
        return None
    code, si, k, huffcode = 0, huffsize[0] if huffsize else 1, 0, []
    while k < len(huffsize):
        while k < len(huffsize) and huffsize[k] == si:
            huffcode.append(code)
            code += 1
            k += 1
        if code >= (1 << si):
            return None
        code <<= 1
        si += 1
    maxcode = np.full(18, -1, np.int64)
    valoffset = np.zeros(18, np.int64)
    p = 0
    for l in range(1, 17):
        if bits[l - 1]:
            valoffset[l] = p - huffcode[p]
            p += bits[l - 1]
            maxcode[l] = huffcode[p - 1]
    maxcode[17] = 0xFFFFF
    lookup = np.zeros(256, np.int16)
    p = 0
    for l in range(1, 9):
        for _ in range(bits[l - 1]):
            base = huffcode[p] << (8 - l)
            lookup[base:base + (1 << (8 - l))] = (l << 8) | vals[p]
            p += 1
    if is_dc and any(v > 15 for v in vals[:len(huffsize)]):
        return None
    t['lookup'], t['maxcode'], t['valoffset'] = lookup, maxcode, valoffset
    t['huffval'][:len(huffsize)] = np.frombuffer(bytes(vals[:len(huffsize)]), np.uint8)
    return t


def parse_header(buf):
    """Walk the markers of `buf` (bytes).  Always returns a Header; height / width are set whenever a frame header was
    read (what Pillow's `size` reports), `device` only for files the device decodes."""
    h = Header()
    buf = bytes(buf)
    n = len(buf)
    if n < 4 or buf[0] != 0xFF or buf[1] != 0xD8:
        return h.host('not a JPEG')
    pos = 2
    qt, dc, ac = {}, {}, {}
    jfif, adobe = False, None
    comps = []
    sof = None
    while True:
        if pos + 4 > n or buf[pos] != 0xFF:
            return h.host('bad marker')
        while pos < n and buf[pos] == 0xFF:
            pos += 1
        if pos + 3 > n:
            return h.host('truncated header')
        m = buf[pos]
        seg = int.from_bytes(buf[pos + 1:pos + 3], 'big')
        body = buf[pos + 3:pos + 1 + seg]
        if seg < 2 or len(body) != seg - 2:
            return h.host('truncated segment')
        pos += 1 + seg
        if 0xC0 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):
            if len(body) < 6:
                return h.host('bad frame header')
            h.height, h.width = int.from_bytes(body[1:3], 'big'), int.from_bytes(body[3:5], 'big')
            if sof is not None:
                return h.host('two frame headers')
            sof = m
            if m not in (0xC0, 0xC1):
                return h.host('not baseline / extended sequential Huffman (SOF%d)' % (m - 0xC0))
            if body[0] != 8:
                return h.host('%d-bit samples' % body[0])
            nc = body[5]
            if len(body) < 6 + 3 * nc:
                return h.host('bad frame header')
            comps = [(body[6 + 3 * i], body[7 + 3 * i] >> 4, body[7 + 3 * i] & 15, body[8 + 3 * i]) for i in range(nc)]
        elif m == 0xC4:                                           # DHT
            p = 0
            while p < len(body):
                if p + 17 > len(body):
                    return h.host('bad DHT')
                tc, th = body[p] >> 4, body[p] & 15
                bits = body[p + 1:p + 17]
                cnt = sum(bits)
                vals = body[p + 17:p + 17 + cnt]
                if tc > 1 or th > 3 or cnt > 256 or len(vals) != cnt:
                    return h.host('bad DHT')
                (dc if tc == 0 else ac)[th] = (bits, vals)
                p += 17 + cnt
        elif m == 0xDB:                                           # DQT
            p = 0
            while p < len(body):
                pq, tq = body[p] >> 4, body[p] & 15
                size = 128 if pq else 64
                if pq > 1 or tq > 3 or p + 1 + size > len(body):
                    return h.host('bad DQT')
                raw = body[p + 1:p + 1 + size]
                qt[tq] = np.frombuffer(raw, '>u2' if pq else np.uint8).astype(np.uint16)
                p += 1 + size
        elif m == 0xDD:                                           # DRI
            if len(body) < 2:
                return h.host('bad DRI')
            h.restart_interval = int.from_bytes(body[:2], 'big')
        elif m == 0xE0:
            if len(body) >= 14 and body[:5] == b'JFIF\x00':        # jdmarker.c examine_app0
                jfif = True
        elif m == 0xEE:
            if len(body) >= 12 and body[:5] == b'Adobe':          # examine_app14
                adobe = body[11]
        elif 0xE1 <= m <= 0xEF or m == 0xFE:
            pass                                                  # APPn / COM
        elif m == 0xDA:                                           # SOS
            break
        else:
            return h.host('marker 0x%02X before the scan' % m)
    if sof is None:
        return h.host('no frame header')
    ns = body[0] if body else 0
    if len(body) < 4 + 2 * ns:
        return h.host('bad scan header')
    sel = [(body[1 + 2 * i], body[2 + 2 * i] >> 4, body[2 + 2 * i] & 15) for i in range(ns)]
    ss, se, ahl = body[1 + 2 * ns], body[2 + 2 * ns], body[3 + 2 * ns]
    nc = len(comps)
    if h.height == 0 or h.width == 0:
        return h.host('empty or DNL-sized frame')
    if nc not in (1, 3):
        return h.host('%d components' % nc)
    if nc == 3:
        ids = [c[0] for c in comps]
        ycc = True                                                # jdapimin.c default_decompress_parms
        if not jfif:
            if adobe is not None:
                ycc = adobe != 0
            elif ids == [82, 71, 66]:
                ycc = False
        if not ycc:
            return h.host('RGB colour space')
        samp = [(c[1], c[2]) for c in comps]
        if samp[1] != (1, 1) or samp[2] != (1, 1) or samp[0] not in ((1, 1), (2, 1), (2, 2)):
            return h.host('sampling %s' % (samp,))
        h.hs, h.vs = samp[0]
    if ns != nc or [s[0] for s in sel] != [c[0] for c in comps]:
        return h.host('not one interleaved scan in frame order')
    if ss != 0 or se != 63 or ahl != 0:
        return h.host('not a sequential scan')
    h.ncomp = nc
    slots = []
    for ci, (cid, td, ta) in enumerate(sel):
        for kind, tid, tables, target in ((0, td, dc, h.dc_tbl), (1, ta, ac, h.ac_tbl)):
            if tid not in tables:
                return h.host('missing Huffman table')
            if (kind, tid) not in slots:
                slots.append((kind, tid))
            target[ci] = slots.index((kind, tid))
    if len(slots) > 4:
        return h.host('more than 4 Huffman tables')
    for kind, tid in slots:
        t = derive_huffman(*(dc if kind == 0 else ac)[tid], is_dc=kind == 0)
        if t is None:
            return h.host('bad Huffman table')
        h.tables.append(t)
    quant = np.zeros((3, 64), np.uint16)
    for ci, c in enumerate(comps):
        if c[3] not in qt:
            return h.host('missing quantisation table')
        quant[ci] = qt[c[3]]
    h.quant = quant
    h.scan_start = pos
    end, marker = scan_end(buf, pos)
    if marker != 0xD9:
        return h.host('the scan is not followed by EOI')
    h.scan_bytes = end - pos                                      # through the EOI marker
    h.device = True
    return h


def mcu_geometry(h):
    """(MCU width, MCU height, MCUs per row, MCU rows, blocks per MCU)."""
    mw, mh = 8 * h.hs, 8 * h.vs
    return mw, mh, -(-h.width // mw), -(-h.height // mh), (1 if h.ncomp == 1 else h.hs * h.vs + 2)


def descriptor(h, crop=None, crop_offset=0):
    """One pf_jpeg_desc for a device-decodable header and a crop window (y, x, h, w) (None: the whole image)."""
    assert h.device
    y, x, ch_, cw_ = crop if crop is not None else (0, 0, h.height, h.width)
    mw, mh, mpr, nrows, _ = mcu_geometry(h)
    # rows / columns of the luma plane and of the chroma planes the crop reads (fancy upsampling reads one neighbour)
    y1, x1 = y + ch_ - 1, x + cw_ - 1
    cy0, cy1 = max(y // h.vs - (h.vs - 1), 0), y1 // h.vs + (h.vs - 1)
    cx0, cx1 = max(x // h.hs - (h.hs - 1), 0), x1 // h.hs + (h.hs - 1)
    ch_rows, ch_cols = -(-h.height // h.vs), -(-h.width // h.hs)
    cy1, cx1 = min(cy1, ch_rows - 1), min(cx1, ch_cols - 1)
    row0 = min(y // mh, cy0 // 8) if h.ncomp == 3 else y // mh
    row1 = max(y1 // mh, cy1 // 8) if h.ncomp == 3 else y1 // mh
    col0 = min(x // mw, cx0 // 8) if h.ncomp == 3 else x // mw
    col1 = max(x1 // mw, cx1 // 8) if h.ncomp == 3 else x1 // mw
    d = np.zeros((), JPEG_DESC)
    d['crop_offset'], d['scan_bytes'] = crop_offset, h.scan_bytes              # scan / workspace offsets: pack()
    d['height'], d['width'], d['ncomp'], d['hs'], d['vs'] = h.height, h.width, h.ncomp, h.hs, h.vs
    d['restart_interval'], d['mcus_per_row'], d['mcu_rows'] = h.restart_interval, mpr, min(row1, nrows - 1) + 1
    d['mcu_row0'], d['mcu_col0'], d['mcu_col1'] = row0, col0, min(col1, mpr - 1)
    d['crop_y'], d['crop_x'], d['crop_h'], d['crop_w'] = y, x, ch_, cw_
    d['dc_tbl'], d['ac_tbl'] = h.dc_tbl, h.ac_tbl
    d['quant'] = h.quant
    for i, t in enumerate(h.tables):
        d['huff'][i] = t
    return d


def workspace_elems(d):
    """int16 coefficients pf_jpeg_decode needs for descriptor d: 64 per block of MCU rows [0, mcu_rows)."""
    bpm = 1 if int(d['ncomp']) == 1 else int(d['hs']) * int(d['vs']) + 2
    return int(d['mcus_per_row']) * int(d['mcu_rows']) * bpm * 64


def scan(h, buf):
    """The entropy-coded segment of a device-decodable file (through its EOI marker)."""
    return buf[h.scan_start:h.scan_start + h.scan_bytes]


def pack(descs, scans):
    """One pf_jpeg_decode batch: descs = pf_jpeg_desc records with their crop_offset set, scans = their files'
    entropy-coded segments.  Returns (descriptor table, uint8 data buffer, workspace int16 elements): the scans back to
    back in order, each image's workspace right after the previous one's."""
    table = np.zeros(len(descs), JPEG_DESC)
    scan_off = ws = 0
    for i, (d, s) in enumerate(zip(descs, scans)):
        table[i] = d
        table[i]['scan_offset'], table[i]['coef_offset'] = scan_off, ws
        scan_off += len(s)
        ws += workspace_elems(d)
    return table, np.frombuffer(bytearray().join(scans), np.uint8), ws
