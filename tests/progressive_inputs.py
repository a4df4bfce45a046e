"""The two inputs that reach the EOBRUN flushes natural pictures do not: a run of 0x7FFF blocks and a
refinement scan whose buffered correction bits pass 937 before any symbol."""
import numpy as np
import scipy.fft

from oracle import jpeg, jpeg_params

CORRECTION_QUALITY = 50


def cap_frame():
  """A flat gray BGR frame of 1536 x 1376 pixels: 33 024 luma blocks whose AC coefficients are all
  zero, so each luma AC scan's EOBRUN reaches 0x7FFF."""
  return np.full((1376, 1536, 3), 117, np.uint8)


def correction_frame(h=128, w=128, seed=0):
  """A gray BGR frame whose luma blocks (quality 50, 4:4:4) have their first twelve AC coefficients
  of magnitude 4 to 7 and the rest zero: after the first scans all of them are known, so the
  refinement scans code no symbol and buffer twelve correction bits per block.  Built by the
  inverse DCT of the dequantized coefficients; blocks that do not requantize to the chosen ones
  (rounding, clipping) are made flat.  -> (frame, the chosen zigzag coefficients [blocks, 64])."""
  rng = np.random.default_rng(seed)
  q = jpeg.quant_tables(CORRECTION_QUALITY)[0]
  rows, cols = h // 8, w // 8
  z = np.zeros((rows * cols, 64), np.int64)
  z[:, 1:13] = rng.integers(4, 8, (rows * cols, 12)) * rng.choice([-1, 1], (rows * cols, 12))
  for _ in range(2):
    nat = np.zeros_like(z)
    nat[:, jpeg.ZIGZAG] = z
    blocks = scipy.fft.idctn((nat * q).reshape(-1, 8, 8).astype(float), axes=(1, 2), norm='ortho') + 128
    px = np.clip(np.rint(blocks), 0, 255).astype(np.uint8)
    img = px.reshape(rows, cols, 8, 8).swapaxes(1, 2).reshape(h, w)
    bgr = np.repeat(img[..., None], 3, axis=2)
    bad = np.any(requantized(bgr) != z, axis=1)
    if not bad.any():
      return bgr, z
    z[bad] = 0
  raise AssertionError('the flat blocks do not requantize to zero')


def requantized(bgr):
  """The luma blocks' zigzag coefficients of a frame whose sides are multiples of 8, at
  CORRECTION_QUALITY and 4:4:4, in raster order."""
  blocks, comp, _, _ = jpeg_params.coefficients(bgr, CORRECTION_QUALITY, CORRECTION_QUALITY, 1, 1)
  return blocks[comp == 0]
