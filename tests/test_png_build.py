"""png.cu compiles for sm_90a, with the Makefile's flags, to kernels with no register spills and no
stack frame, as DESIGN.md reports them."""
import os
import re
import subprocess
import tempfile

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'squeezedet_b200',
                    'csrc')
KERNELS = ('filter_kernel', 'mark_kernel', 'seg_scan_kernel', 'count_kernel', 'emit_kernel',
           'tree_kernel', 'frame_kernel', 'pack_kernel', 'idat_kernel')


def makefile_flags():
  """NVCC and NVCCFLAGS of the Makefile, $(ARCH) expanded and $(EXTRA) empty."""
  text = open(os.path.join(CSRC, 'Makefile')).read().replace('\\\n', ' ')
  var = dict(re.findall(r'^(\w+)\s*[?:]?=\s*(.*)$', text, re.M))
  flags = var['NVCCFLAGS'].replace('$(ARCH)', var['ARCH']).replace('$(EXTRA)', '')
  return os.environ.get('NVCC', var['NVCC']), flags.split()


def test_png_kernels_do_not_spill():
  nvcc, flags = makefile_flags()
  with tempfile.TemporaryDirectory() as tmp:
    r = subprocess.run([nvcc] + flags + ['-Xptxas', '-v', '-c', 'png.cu', '-o',
                                         os.path.join(tmp, 'png.o')],
                       cwd=CSRC, capture_output=True, text=True, check=True)
  report = {}
  name = None
  for line in r.stderr.splitlines():
    m = re.search(r"Function properties for (\S+)", line)
    if m:
      name = m.group(1)
    m = re.search(r'(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads', line)
    if m and name:
      report[name] = tuple(int(v) for v in m.groups())
      name = None
  kernels = {n: v for n, v in report.items() if any(k in n for k in KERNELS)}
  assert all(any(k in n for n in kernels) for k in KERNELS), sorted(report)
  assert all(v == (0, 0, 0) for v in kernels.values()), kernels
