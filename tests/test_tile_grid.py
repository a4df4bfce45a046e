"""utils.util.tile_grid: the fewest evenly spaced tiles per axis that cover a frame with at least
min_overlap pixels of overlap, the last flush with the far edge."""
import pytest

from squeezedet_b200.utils.util import tile_grid


def axis_positions(grid, coord):
  return sorted({t[coord] for t in grid})


def check_axis(pos, size, frame, min_overlap):
  assert pos[0] == 0 and pos[-1] + size == frame                 # covers, last flush
  for a, b in zip(pos, pos[1:]):
    assert b > a and a + size - b >= min_overlap                  # overlap at least min_overlap
  if len(pos) > 1:                                                # one tile fewer cannot do it
    k = len(pos) - 1
    assert k == 1 or (k - 1) * (size - min_overlap) + size < frame
  steps = [b - a for a, b in zip(pos, pos[1:])]
  assert not steps or max(steps) - min(steps) <= 1                # evenly spaced


def test_1080p_kitti_tiles():
  grid = tile_grid(1920, 1080, 1242, 375, 128)
  assert len(grid) == 8
  assert axis_positions(grid, 0) == [0, 678]
  assert axis_positions(grid, 1) == [0, 235, 470, 705]
  assert all(t[2:] == (1242, 375) for t in grid)
  assert grid[:2] == [(0, 0, 1242, 375), (678, 0, 1242, 375)]   # row-major


@pytest.mark.parametrize('frame_w,frame_h,tile_w,tile_h,overlap', [
    (1920, 1080, 1242, 375, 128), (3840, 2160, 1242, 375, 0), (3840, 2160, 1248, 384, 200),
    (1243, 376, 1242, 375, 0), (2484, 750, 1242, 375, 0), (2485, 751, 1242, 375, 1),
    (5000, 377, 1242, 375, 374), (1300, 700, 1242, 375, 64)])
def test_cover_and_overlap(frame_w, frame_h, tile_w, tile_h, overlap):
  grid = tile_grid(frame_w, frame_h, tile_w, tile_h, overlap)
  xs, ys = axis_positions(grid, 0), axis_positions(grid, 1)
  assert len(grid) == len(xs) * len(ys)
  check_axis(xs, tile_w, frame_w, overlap)
  check_axis(ys, tile_h, frame_h, overlap)


def test_exact_fit_is_one_tile():
  assert tile_grid(1242, 375, 1242, 375, 128) == [(0, 0, 1242, 375)]


def test_frame_smaller_than_a_tile():
  assert tile_grid(640, 360, 1242, 375, 128) == [(0, 0, 640, 360)]
  grid = tile_grid(1920, 300, 1242, 375, 128)                    # short on one axis only
  assert grid == [(0, 0, 1242, 300), (678, 0, 1242, 300)]
  assert tile_grid(1000, 1080, 1242, 375, 128)[0] == (0, 0, 1000, 375)


def test_bad_arguments():
  with pytest.raises(ValueError):
    tile_grid(1920, 1080, 1242, 375, 375)                         # overlap as tall as a tile
  with pytest.raises(ValueError):
    tile_grid(1920, 1080, 1242, 375, -1)
  with pytest.raises(ValueError):
    tile_grid(0, 1080, 1242, 375, 128)
