"""Every entry point of the C ABI has a kernel test: some tests/test_*_gpu.py calls it directly, as `ops.<name>(` or
`ops.lib.tfx_<name>(`.  Whole-model parity runs most kernels too, but at loose tolerances and small shapes; a kernel that is
only reached that way can be subtly wrong without any test failing.  Reads the test sources as text; needs no GPU."""
import pathlib
import re

from transfusion_pytorch_b200 import _lib

TESTS = pathlib.Path(__file__).resolve().parent

# entry points that are not kernels, each with the reason it needs no direct kernel test
EXEMPT = {
    'tfx_init': 'configuration: checks the device, launches nothing',
    'tfx_version': 'returns a constant',
    'tfx_last_error': 'returns the thread-local error message',
}


def _called(name, sources):
    short = name[len('tfx_'):]
    pat = re.compile(r'\bops\.' + re.escape(short) + r'\(|\bops\.lib\.' + re.escape(name) + r'\(')
    return any(pat.search(src) for src in sources)


def test_every_entry_point_has_a_kernel_test():
    sources = [p.read_text() for p in sorted(TESTS.glob('test_*_gpu.py'))]
    assert sources
    names = sorted(set(_lib.SIGNATURES) | set(_lib.EXPORTED))
    missing = [n for n in names if n not in EXEMPT and not _called(n, sources)]
    assert not missing, f'entry points with no direct call in tests/test_*_gpu.py: {missing}'


def test_exemptions_name_real_entry_points():
    names = set(_lib.SIGNATURES) | set(_lib.EXPORTED)
    assert set(EXEMPT) <= names, sorted(set(EXEMPT) - names)
    assert all(reason.strip() for reason in EXEMPT.values())
