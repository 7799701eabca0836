"""Plan tables and the plan-device check of libkapre_b200, read from ``csrc/kapre_b200.cu``.

Every plan holds its constant device tables in one block, built by ``KbTableUpload`` and owned by a ``KbTables``
member that frees it when the plan is deleted.  A table added to a plan can then not be left out of a hand-kept list
of frees.  Every entry point that takes a plan checks the plan's device through ``kb_check_device``, so no entry can
launch kernels on one device that read tables made on another.  The source is checked here: one ``cudaMalloc`` and one
``cudaMemcpy``, both in the upload, one ``cudaFree``, in ``KbTables``, and one copy of the device-mismatch message, in
``kb_check_device``."""
import os
import re

from test_launch_sites import _body_span, _code, _sites

SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'kapre_b200', 'csrc', 'kapre_b200.cu')


def _one_site_inside(code, pattern, head, what):
    sites = _sites(code, pattern)
    assert len(sites) == 1, '%s appears %d times in %s' % (what, len(sites), SRC)
    lo, hi = _body_span(code, head)
    assert lo <= sites[0] < hi, '%s is outside %r' % (what, head)


def test_tables_are_allocated_copied_and_freed_in_one_place():
    code = _code()
    _one_site_inside(code, r'\bcudaMalloc\s*\(', r'\bclass\s+KbTableUpload\b', 'cudaMalloc')
    _one_site_inside(code, r'\bcudaMemcpy\s*\(', r'\bclass\s+KbTableUpload\b', 'cudaMemcpy')
    _one_site_inside(code, r'\bcudaFree\s*\(', r'\bstruct\s+KbTables\b', 'cudaFree')
    assert not _sites(code, r'\bkb_upload\b'), 'kb_upload is back: upload plan tables through KbTableUpload'


def test_one_device_check():
    text = open(SRC).read()   # the message is a string literal, which _code() blanks out
    sites = [m.start() for m in re.finditer(r'was created on device', text)]
    assert len(sites) == 1, 'the device-mismatch message appears %d times; call kb_check_device' % len(sites)
    lo, hi = _body_span(_code(), r'static\s+int\s+kb_check_device\s*\(')
    assert lo <= sites[0] < hi, 'the device-mismatch message is outside kb_check_device'
