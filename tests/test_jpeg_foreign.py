"""Files other encoders write, on the host: the test writer's transcodes decode (in cv2) to their
sources' pixels, the oracle matches cv2 on them, and sqdet_jpeg_parse agrees with the oracle's
parse; EXIF orientation is read as cv2 reads it; files refused by design are refused with their
reason, by sqdet_jpeg_parse and sqdet_decode_jpeg alike."""
import ctypes as C

import cv2
import numpy as np
import pytest

from oracle import jpeg_decode as D
from squeezedet_b200 import _lib
from squeezedet_b200.jpeg import jpeg_info

import jpeg_corpus as J
import jpeg_writer as W


@pytest.fixture(scope='module')
def foreign():
  return J.foreign()


def test_writer_keeps_pixels(foreign):
  for name, f, src in foreign:
    want = J.imdecode(src)
    got = J.imdecode(f)
    assert got is not None and got.shape == want.shape and np.array_equal(got, want), name


def test_oracle_is_cv2_on_foreign(foreign):
  for name, f, _ in foreign:
    assert np.array_equal(D.decode(f), J.imdecode(f)), name


def test_parse_agrees_with_oracle(foreign):
  for name, f, _ in foreign:
    i, p = jpeg_info(f), D.parse(f)
    assert i['supported'], (name, i['reason_text'])
    assert (i['height'], i['width']) == p.out_hw, name
    assert (i['coded_height'], i['coded_width']) == (p.height, p.width), name
    assert (i['h_samp'], i['v_samp']) == ((p.comps[0].h, p.comps[0].v) if len(p.comps) == 3 else (1, 1)), name
    assert i['restart_interval'] == p.restart and i['scan_offset'] == p.scan, name
    assert i['orientation'] == p.orientation == 1, name


def test_variants_reach_what_they_name(foreign):
  # each setting shows up in the bytes: tables on selectors 2 and 3, a third quantization table,
  # codes of 15 and 16 bits, 256-symbol tables, fill bytes before RSTn, SOF1
  by = {n: D.parse(f) for n, f, _ in foreign}
  some = lambda key, pred: any(pred(p) for n, p in by.items() if n.endswith(key))
  assert some('chroma on 2,3', lambda p: [(c.td, c.ta) for c in p.comps] == [(0, 0), (2, 3), (2, 3)])
  assert some('Cb, Cr apart', lambda p: len({(c.td, c.ta) for c in p.comps}) == 3)
  assert some('quant 3, 0, 2', lambda p: [c.tq for c in p.comps] == [3, 0, 2])
  assert some(', skewed', lambda p: p.ac[p.comps[0].ta][0][14:] == [1, 1])
  assert some('full 256', lambda p: len(p.ac[p.comps[0].ta][1]) == 256 and len(p.dc[p.comps[0].td][1]) == 16)
  halved = [n for n, p in by.items() if n.endswith('Cr quant halved') and not np.array_equal(p.qt[1], p.qt[2])]
  assert len(halved) >= 3, halved
  assert all(b'\xff\xff\xff\xff\xd0' in f for n, f, _ in foreign if n.endswith('rst 2 fill bytes'))
  assert all(b'\xff\xc1' in f[:by[n].scan] for n, f, _ in foreign if n.endswith('sof1'))


def test_optimal_tables_are_cv2s():
  # the writer's jpeg_gen_optimal_table builds from a file's symbol counts the tables cv2's
  # optimizing encoder wrote for it
  rng = np.random.default_rng(3)
  for kind, samp in (('noise', 0x111111), ('smooth', 0x221111), ('check', 0x211111)):
    f = J.encode(J.content(kind, 40, 64, 3, rng), cv2.IMWRITE_JPEG_OPTIMIZE, 1,
                 cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp)
    info, grids = W.source(f)
    freq = {}
    for iv in W.scan_symbols(info, grids, range(3), 0):
      for ci, syms in iv:
        for is_ac, s, _, _ in syms:
          key = (is_ac, (info.comps[ci].ta if is_ac else info.comps[ci].td))
          freq.setdefault(key, {})
          freq[key][s] = freq[key].get(s, 0) + 1
    for (is_ac, tid), fr in freq.items():
      bits, vals = (info.ac if is_ac else info.dc)[tid]
      assert W.optimal_table(fr) == (list(bits), list(vals)), (kind, is_ac, tid)
    g = W.write(info, grids, tables='optimal', pack='joint')
    assert g[D.parse(g).scan:] == f[info.scan:], kind


@pytest.mark.parametrize('row', range(len(J.exif_variants())))
def test_exif_orientation_as_cv2(row):
  name, f, want = J.exif_variants()[row]
  first = J.exif_variants()[0][1]                     # its Exif APP1 is the first segment
  plain = J.imdecode(first[:2] + first[4 + int.from_bytes(first[4:6], 'big'):])
  assert np.array_equal(J.imdecode(f), D.orient(plain, want)), '%s: cv2 no longer applies %d' % (name, want)
  assert D.parse(f).orientation == want, name
  assert np.array_equal(D.decode(f), J.imdecode(f)), name
  i = jpeg_info(f)
  assert i['orientation'] == want, name
  assert (i['height'], i['width']) == ((21, 13) if want >= 5 else (13, 21)), name


def test_refused_by_design():
  lib = _lib.load()
  for name, f, reason, cv2_decodes in J.refused():
    assert (J.imdecode(f) is not None) == cv2_decodes, name
    i = jpeg_info(f)
    assert not i['supported'] and i['reason'] == reason, (name, i)
    with pytest.raises(D.Unsupported) as e:
      D.parse(f)
    assert e.value.reason == reason, name
    buf = C.create_string_buffer(f, len(f))
    fake = 1 << 40                                    # never dereferenced: the refusal comes first
    rc = lib.sqdet_decode_jpeg(1, (C.c_void_p * 1)(C.addressof(buf)), (C.c_int64 * 1)(len(f)),
                               (C.c_void_p * 1)(fake), (C.c_int64 * 1)(3 * 64), fake, 1 << 40,
                               fake, 1 << 40, fake, None)
    assert rc == -3, name
    assert D.REASONS[reason].encode() in lib.sqdet_last_error(), name


@pytest.fixture(scope='module')
def camera():
  return J.camera()


def test_camera_files_parse(camera):
  want = {'4000x3000 q92 s221111 exif 6': ((4000, 3000), 6, (2, 2), 0),
          '3000x4000 q95 s211111 rst row exif 8': ((3000, 4000), 8, (2, 1), 3000 // 16 + 1),
          '4032x3024 noise q100 s111111': ((3024, 4032), 1, (1, 1), 0),
          '1x8191': ((1, 8191), 1, (2, 2), 0), '8191x1': ((8191, 1), 1, (2, 2), 0)}
  for name, f in camera:
    i = jpeg_info(f)
    hw, o, samp, rst = want[name]
    assert i['supported'], name
    assert ((i['height'], i['width']), i['orientation'], (i['h_samp'], i['v_samp']),
            i['restart_interval']) == (hw, o, samp, rst), name
    assert J.imdecode(f).shape == hw + (3,), name
    p = D.parse(f)
    assert p.out_hw == hw and p.scan == i['scan_offset'], name
  assert len(camera[2][1]) > 40 << 20


def test_oracle_on_a_camera_file(camera):
  f = dict(camera)['8191x1']
  assert np.array_equal(D.decode(f), J.imdecode(f))
