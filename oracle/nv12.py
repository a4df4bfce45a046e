"""CPU restatement of the NV12 -> BGR colour conversion in front of the NV12 device-frames path
(sqdet_forward_frames_nv12) — test infrastructure, like the rest of oracle/.

The reference stack converts with ``cv2.cvtColor(nv12, cv2.COLOR_YUV2BGR_NV12)``: OpenCV's BT.601
limited-range fixed-point conversion (ITUR_BT_601_* constants, 20 fraction bits), restated here
operation for operation and PINNED bitwise against the installed cv2 (tests/test_oracle_nv12.py).
It is not FFmpeg's swscale inside ``cv2.VideoCapture``, whose rounding differs."""
import numpy as np


def nv12_to_bgr(luma, chroma):
  """cv2.cvtColor(nv12, cv2.COLOR_YUV2BGR_NV12) for luma [H, W] and interleaved U,V chroma
  [H/2, W] (uint8, H and W even) -> uint8 BGR [H, W, 3]."""
  y = np.asarray(luma, np.uint8).astype(np.int32)
  uv = np.asarray(chroma, np.uint8).astype(np.int32)
  h, w = y.shape
  assert h % 2 == 0 and w % 2 == 0 and uv.shape == (h // 2, w), (y.shape, uv.shape)
  u = np.repeat(np.repeat(uv[:, 0::2], 2, axis=0), 2, axis=1) - 128
  v = np.repeat(np.repeat(uv[:, 1::2], 2, axis=0), 2, axis=1) - 128
  yy = np.maximum(y - 16, 0) * 1220542 + (1 << 19)
  sat = lambda x: np.clip(x >> 20, 0, 255).astype(np.uint8)  # noqa: E731
  return np.stack([sat(yy + 2116026 * u), sat(yy - 852492 * v - 409993 * u),
                   sat(yy + 1673527 * v)], axis=-1)
