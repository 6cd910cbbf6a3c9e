"""CPU guard on the machine code of the CLIP preprocessing kernels (csrc/clip_preprocess.cu: clip_resize_1,
clip_resize_2_sample), read from the built library with cuobjdump: integer resize passes, no fp16 twin, no local
memory, at the register counts of DESIGN.md section 3."""
import re
import shutil
import subprocess

import pytest


def test_clip_kernels_registers_and_no_local_memory():
    if shutil.which('cuobjdump') is None:
        pytest.skip('cuobjdump unavailable')
    from gpt4roi_b200 import build, lib
    build.build()
    res = subprocess.run(['cuobjdump', '-res-usage', lib.LIB_PATH], capture_output=True, text=True)
    if res.returncode != 0:
        pytest.skip('cuobjdump unavailable')
    found = re.findall(r'Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)', res.stdout)
    usage = {n: (int(r), int(s), int(l)) for n, r, s, l in found if 'clip_resize_' in n}
    assert len(usage) == 2, usage                     # no fp16 twin: integer resize, one instance each
    for name, (regs, stack, local) in usage.items():
        want = 32 if 'clip_resize_1' in name else 48
        assert regs == want and stack == 0 and local == 0, (name, regs, stack, local)
        out = subprocess.run(['cuobjdump', '-sass', '-fun', name, lib.LIB_PATH], capture_output=True, text=True,
                             check=True).stdout
        assert not re.findall(r'\b(?:STL|LDL)(?:\.\w+)*\s', out), name
