"""JPEG files of every colour space and sampling cv2.imdecode reads, for the any-layout decoder's
tests: CMYK and YCCK (4 components), RGB-coded files (Adobe transform 0, or ids 'R', 'G', 'B'
without JFIF), and samplings other encoders write and cv2's never does.

make() codes smooth random planes laid out for any sampling straight into coefficients (an
orthonormal 8 x 8 DCT, quantized) and writes them with jpeg_writer, so any layout can be built;
with a scan script it writes them as SOF2 through progressive_writer.  Pillow writes the CMYK and
keep_rgb files other software meets."""
import io
from unittest import mock

import numpy as np
from scipy.fft import dctn

from oracle import jpeg_decode as D
from oracle import jpeg_decode_layouts as L

import jpeg_corpus as J
import jpeg_writer as W
import progressive_writer as PW

YCC_IDS, RGB_IDS = (1, 2, 3), (82, 71, 66)
CMYK_IDS = (67, 77, 89, 75)
JFIF = W.segment(0xE0, b'JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00')


def adobe(transform):
  """An APP14 Adobe segment with this colour transform."""
  return W.segment(0xEE, b'Adobe\x00\x64\x00\x00\x00\x00' + bytes([transform]))


def quant(scale):
  """A quantization table (natural order) growing with frequency, times scale, in [1, 255]."""
  u, v = np.mgrid[:8, :8]
  return np.clip(np.round((2 + 2 * (u + v)) * scale), 1, 255).astype(np.uint16).ravel()


def make(h, w, sampling, ids=None, markers=(), scale=1.0, restart=0, seed=0, script=None):
  """A sequential h x w file of len(sampling) components with these (h, v) factors, with
  `markers` (segments such as JFIF or adobe(t)) after SOI; with a scan script, progressive (SOF2,
  progressive_writer's scans; () for SCRIPT or SCRIPT4).  Component 0 takes table 0, the others table 1, each from
  quant(scale)."""
  rng = np.random.default_rng(seed)
  nc = len(sampling)
  ids = ids or (CMYK_IDS if nc == 4 else YCC_IDS[:nc])
  hmax, vmax = (max(s[0] for s in sampling), max(s[1] for s in sampling)) if nc > 1 else (1, 1)
  mcols, mrows = -(-w // (8 * hmax)), -(-h // (8 * vmax))
  q = {0: quant(scale), 1: quant(1.5 * scale)}
  grids = []
  for k, (ch, cv) in enumerate(sampling):
    bh, bw = (mrows * cv, mcols * ch) if nc > 1 else (mrows, mcols)
    px = J.content('smooth', bh * 8, bw * 8, 1, rng)[..., 0].astype(np.float64) - 128
    coef = dctn(px.reshape(bh, 8, bw, 8).transpose(0, 2, 1, 3), axes=(2, 3), norm='ortho')
    grids.append(np.round(coef.reshape(bh, bw, 64) / q[min(k, 1)]).astype(np.int32))
  comps = [D.Component(ids[k], ch, cv, min(k, 1)) for k, (ch, cv) in enumerate(sampling)]
  info = D.Info(h, w, comps, q, {}, {}, hmax=hmax, vmax=vmax)
  if script is None:
    return W.write(info, grids, tables='optimal', restart=restart, before=tuple(markers), jfif=False)
  # progressive_writer transcodes a file it parses; these coefficients go to it directly, and its
  # JFIF APP0 gives way to `markers`
  with mock.patch.object(PW, 'source', lambda _: (info, grids)), \
       mock.patch.object(PW, '_scan_items', _scan_items):
    p = PW.write(b'', [sc for sc in script or (SCRIPT4 if nc == 4 else SCRIPT) if min(sc[0]) < nc])
  return b'\xff\xd8' + b''.join(markers) + p[2 + len(JFIF):]


# complete scripts (progressive_writer drops the components a file lacks): interleaved DC scans,
# or one DC scan per component where an interleaved MCU would pass 10 blocks
SCRIPT = [((0, 1, 2), 0, 0, 0, 1), ((0,), 1, 5, 0, 0), ((0,), 6, 63, 0, 0), ((2,), 1, 63, 0, 1),
          ((1,), 1, 63, 0, 0), ((2,), 1, 63, 1, 0), ((0, 1, 2), 0, 0, 1, 0)]
SCRIPT4 = SCRIPT[:1] + [((3,), 0, 0, 0, 1)] + SCRIPT[1:] + [((3,), 1, 63, 0, 0), ((3,), 0, 0, 1, 0)]
SCRIPT_SPLIT_DC = [((c,), 0, 0, 0, 0) for c in range(4)] + [((c,), 1, 63, 0, 0) for c in range(4)]


def _scan_items(rows, ucomp, dummy, per, scan, restart, counts):
  """oracle.jpeg_progressive's scan coder, which keeps DC predictors for components 0..2 and codes
  component 0 with table 0 and the others with table 1: component 3 takes the place of one of 1
  and 2 that the scan lacks."""
  free = [c for c in (2, 1) if c not in scan[0]]
  remap = np.array([0, 1, 2, free[0] if free else 3])
  return _scan_items.coder(rows, remap[np.asarray(ucomp)], dummy, per, scan, restart, counts)


_scan_items.coder = PW._scan_items


def pillow(img, mode, **kw):
  """Pillow's JPEG of uint8 img [h, w, c] in `mode` ('CMYK' or 'RGB')."""
  from PIL import Image
  buf = io.BytesIO()
  Image.fromarray(img, mode).save(buf, 'JPEG', **kw)
  return buf.getvalue()


# (h, v) per component of samplings cv2's encoder never writes; every one has integral ratios and
# at most 10 blocks per MCU
ODD_SAMPLINGS = {
    'cb 2x2 cr 1x1': [(2, 2), (2, 2), (1, 1)],
    'cb 2x1 cr 1x2': [(2, 2), (2, 1), (1, 2)],
    'chroma finer than luma': [(1, 1), (2, 2), (2, 2)],
    'luma 1x1 chroma 2x1 1x2': [(1, 1), (2, 1), (1, 2)],
    'h3': [(3, 1), (1, 1), (1, 1)],
    'v3': [(1, 3), (1, 1), (1, 1)],
    'h3 v2': [(3, 2), (1, 1), (1, 1)],
    'h4 v2 (10 blocks)': [(4, 2), (1, 1), (1, 1)],
    'v4': [(1, 4), (1, 1), (1, 1)],
    'h4 cb h2': [(4, 1), (2, 1), (1, 1)],
    'h1 v4 cb v2': [(1, 4), (1, 2), (1, 1)],
}
# what libjpeg rejects: cv2.imdecode returns None
BAD_SAMPLINGS = {
    'fractional h 3 / 2': [(3, 1), (2, 1), (1, 1)],
    'fractional v 4 / 3': [(1, 4), (1, 3), (1, 1)],
    '11 blocks': [(3, 3), (1, 1), (1, 1)],
    'cmyk 13 blocks': [(2, 2), (2, 2), (2, 2), (1, 1)],
}


def corpus(seed=0):
  """[(name, file)] of files the any-layout decoder decodes, sequential and progressive."""
  rng = np.random.default_rng(seed)
  out = []
  for q in (30, 75, 95, 100):
    for sub in (0, 2):
      img = J.content('smooth', 37 + q % 7, 45 + sub, 4, rng)
      out.append(('pillow cmyk q%d s%d' % (q, sub), pillow(img, 'CMYK', quality=q, subsampling=sub)))
  # Pillow writes keep_rgb files at 4:4:4 only
  out.append(('pillow keep_rgb', pillow(J.content('smooth', 29, 51, 3, rng), 'RGB', quality=90, keep_rgb=True)))
  c444, c420 = [(1, 1)] * 4, [(2, 2), (1, 1), (1, 1), (2, 2)]
  specs = [('cmyk no app14', dict(h=27, w=35, sampling=c444)),
           ('cmyk adobe 0 (2,2,1,1,1,1,2,2: 10 blocks)', dict(h=41, w=38, sampling=c420, markers=[adobe(0)])),
           ('ycck', dict(h=33, w=30, sampling=c444, markers=[adobe(2)])),
           ('ycck subsampled', dict(h=35, w=47, sampling=[(2, 2), (1, 1), (1, 1), (1, 1)], markers=[adobe(2)])),
           ('4 components adobe 1', dict(h=19, w=22, sampling=c444, markers=[adobe(1)])),
           ('4 components adobe 7', dict(h=18, w=25, sampling=[(1, 2), (1, 1), (1, 1), (1, 2)], markers=[adobe(7)])),
           ('3 components adobe 2', dict(h=21, w=30, sampling=[(2, 1), (1, 1), (1, 1)], markers=[adobe(2)])),
           ('rgb adobe 0', dict(h=25, w=31, sampling=[(1, 1)] * 3, markers=[adobe(0)])),
           ('rgb adobe 0 subsampled', dict(h=26, w=33, sampling=[(2, 2), (1, 1), (1, 1)], markers=[adobe(0)])),
           ('rgb ids', dict(h=23, w=29, sampling=[(1, 1)] * 3, ids=RGB_IDS)),
           ('rgb ids subsampled', dict(h=23, w=29, sampling=[(2, 1), (1, 1), (1, 1)], ids=RGB_IDS)),
           ('rgb ids after jfif: ycc', dict(h=23, w=29, sampling=[(1, 1)] * 3, ids=RGB_IDS, markers=[JFIF])),
           ('rgb ids after adobe 1: ycc', dict(h=23, w=29, sampling=[(1, 1)] * 3, ids=RGB_IDS, markers=[adobe(1)])),
           ('rgb adobe 0 restart 3', dict(h=40, w=50, sampling=[(1, 2), (1, 1), (1, 1)], markers=[adobe(0)], restart=3))]
  specs += [(name, dict(h=35 + k, w=43 + 2 * k, sampling=samp, markers=[JFIF]))
            for k, (name, samp) in enumerate(ODD_SAMPLINGS.items())]
  # 4:2:0 chroma 1, 2 and 3 samples wide and high, around the fancy upsampling's width threshold
  for w in (1, 2, 3, 4, 5, 6):
    specs.append(('cmyk 4:2:0 %dx%d' % (w, w), dict(h=w, w=w, sampling=c420)))
    specs.append(('chroma finer %dx%d' % (w + 1, w), dict(h=w + 1, w=w, sampling=[(1, 1), (2, 2), (2, 1)])))
  out += [(name, make(seed=seed + k, **kw)) for k, (name, kw) in enumerate(specs)]
  out += [(name + ' progressive', make(seed=seed + k, script=(), **kw))
          for k, (name, kw) in enumerate(specs) if k % 2 == 0 and 'restart' not in kw]
  out.append(('h4 v2 progressive, one DC scan per component',
              make(30, 70, ODD_SAMPLINGS['h4 v2 (10 blocks)'], markers=[JFIF], seed=seed, script=SCRIPT_SPLIT_DC)))
  return out


def wide_progressive(seed=0):
  """A progressive CMYK file of 13 blocks per MCU with no interleaved scan: cv2 decodes it, the
  any-layout decoder refuses it as SAMPLING."""
  return make(30, 40, BAD_SAMPLINGS['cmyk 13 blocks'], seed=seed, script=SCRIPT_SPLIT_DC)


def remainders(sampling, markers=(), seed=0):
  """[(name, file)]: every remainder of the width modulo 8 * hmax and of the height modulo 8 *
  vmax, paired off, at one block row or column past a multiple and past two."""
  hmax, vmax = max(s[0] for s in sampling), max(s[1] for s in sampling)
  mw, mh = 8 * hmax, 8 * vmax
  n = max(mw, mh)
  return [('%dx%d' % (mh + k % mh + 1, mw + k % mw + 1),
           make(mh + k % mh + 1, mw + k % mw + 1, sampling, markers=markers, seed=seed + k))
          for k in range(n)]


def refused(seed=0):
  """[(name, file, reason)] that the any-layout decoder refuses and cv2.imdecode returns None for."""
  out = [(name, make(20, 30, samp, seed=seed + k), L.BAD_SAMPLING)
         for k, (name, samp) in enumerate(BAD_SAMPLINGS.items())]
  out.append(('2 components', make(16, 16, [(1, 1), (1, 1)], ids=(1, 2), seed=seed + 10), D.COMPONENTS))
  out.append(('5 components', make(16, 16, [(1, 1)] * 5, ids=(1, 2, 3, 4, 5), seed=seed + 11), D.COMPONENTS))
  # a progressive frame libjpeg accepts, with an interleaved DC scan of 11 blocks
  out.append(('progressive 11-block DC scan', make(24, 40, BAD_SAMPLINGS['11 blocks'], markers=[JFIF],
                                                   seed=seed + 12, script=()), L.BAD_SAMPLING))
  return out
