"""Every kernel launch of libkapre_b200 goes through one helper, ``kb_launch`` in ``csrc/kapre_b200.cu``.

That helper is where the launch count (``kapre_launch_count``) is bumped and where the launches that the profiler
times (``kapre_profile_read``, the kernel time of ``bench.py``) are bracketed with events.  A launch written anywhere
else would compile and run, but silently miscount launches or change what the benchmark times, so the source is
checked here: one ``cudaLaunchKernelEx``, no triple-chevron launch, one ``g_launches++`` and one ``KbProfScope``,
all inside ``kb_launch``."""
import os
import re

SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'kapre_b200', 'csrc', 'kapre_b200.cu')


def _code():
    """The source with comments and string literals blanked out (same length, so offsets still line up)."""
    text = open(SRC).read()
    pat = re.compile(r'//[^\n]*|/\*.*?\*/|"(?:\\.|[^"\\\n])*"', re.S)
    return pat.sub(lambda m: ' ' * len(m.group(0)), text)


def _body_span(code, head):
    """[start, end) of the brace-delimited body of the first definition matching the regex `head`."""
    m = re.search(head, code)
    assert m, 'no definition matching %r in %s' % (head, SRC)
    start = code.index('{', m.end())
    depth = 0
    for i in range(start, len(code)):
        if code[i] == '{':
            depth += 1
        elif code[i] == '}':
            depth -= 1
            if depth == 0:
                return start, i + 1
    raise AssertionError('unbalanced braces after %r' % head)


def _sites(code, pattern):
    return [m.start() for m in re.finditer(pattern, code)]


def test_one_launch_site_inside_kb_launch():
    code = _code()
    lo, hi = _body_span(code, r'static\s+int\s+kb_launch\s*\(')
    checks = {
        'cudaLaunchKernelEx': r'\bcudaLaunchKernelEx\s*\(',
        'g_launches++': r'\bg_launches\s*\+\+',
        'KbProfScope construction': r'\bKbProfScope\s+\w+\s*[({]',
    }
    for name, pattern in checks.items():
        sites = _sites(code, pattern)
        assert len(sites) == 1, '%s appears %d times; every launch must go through kb_launch' % (name, len(sites))
        assert lo <= sites[0] < hi, '%s is outside kb_launch' % name
    assert not _sites(code, r'<<<'), 'triple-chevron launch outside kb_launch'
    # no other way of bumping the count or launching
    assert not _sites(code, r'\bg_launches\s*(\+=|=[^=])'), 'g_launches changed outside kb_launch'
    assert not _sites(code, r'\bcudaLaunch(Kernel|CooperativeKernel)\s*\('), 'launch API called outside kb_launch'
