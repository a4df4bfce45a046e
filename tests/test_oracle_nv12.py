"""Pins oracle.nv12.nv12_to_bgr bitwise against the installed cv2's
cvtColor(COLOR_YUV2BGR_NV12), the conversion the NV12 device-frames path reproduces."""
import numpy as np
import pytest

from oracle import nv12 as oracle_nv12

cv2 = pytest.importorskip('cv2')

SHAPES = [(1080, 1920), (376, 1242), (370, 1224), (2, 2), (2, 4), (10, 6)]


def nv12(h, w, seed, edges):
  """(luma [h, w], chroma [h/2, w]); with `edges`, every byte at a clamping edge: Y in 0..16 or
  235..255, U and V at 0 or 255."""
  rng = np.random.default_rng(seed)
  if not edges:
    return (rng.integers(0, 256, (h, w), dtype=np.uint8),
            rng.integers(0, 256, (h // 2, w), dtype=np.uint8))
  y_edge = np.concatenate([np.arange(0, 17), np.arange(235, 256)]).astype(np.uint8)
  return rng.choice(y_edge, (h, w)), rng.choice(np.array([0, 255], np.uint8), (h // 2, w))


@pytest.mark.parametrize('edges', [False, True], ids=['random', 'edges'])
@pytest.mark.parametrize('h,w', SHAPES)
def test_nv12_to_bgr_bitwise_cv2(h, w, edges):
  luma, chroma = nv12(h, w, h * 31 + w + edges, edges)
  want = cv2.cvtColor(np.concatenate([luma, chroma]), cv2.COLOR_YUV2BGR_NV12)
  got = oracle_nv12.nv12_to_bgr(luma, chroma)
  assert got.dtype == np.uint8 and got.shape == (h, w, 3)
  np.testing.assert_array_equal(got, want)


def test_nv12_to_bgr_every_yuv_triple():
  """All 256^3 (Y, U, V) triples in one 4096 x 4096 frame: 2x2 block b (row-major over the
  2048 x 2048 blocks) has chroma sample b % 65536 and luma 4 * (b // 65536) + {0, 1, 2, 3}."""
  b = np.arange(2048 * 2048).reshape(2048, 2048)
  uv = b % 65536
  chroma = np.stack([uv >> 8, uv & 255], axis=-1).reshape(2048, 4096).astype(np.uint8)
  base = 4 * (b // 65536)
  luma = np.empty((4096, 4096), np.uint8)
  for k, (r, c) in enumerate([(0, 0), (0, 1), (1, 0), (1, 1)]):
    luma[r::2, c::2] = base + k
  want = cv2.cvtColor(np.concatenate([luma, chroma]), cv2.COLOR_YUV2BGR_NV12)
  np.testing.assert_array_equal(oracle_nv12.nv12_to_bgr(luma, chroma), want)
