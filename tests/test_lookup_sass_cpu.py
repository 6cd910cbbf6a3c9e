"""CPU guard on the machine code of the prompt-lookup kernel (csrc/lookup.cu: g4r_lookup_step / g4r_lookup_draft), read
from the built library with cuobjdump: one integer-only instance, 32 registers (DESIGN.md section 3), no local memory."""
import re
import shutil
import subprocess

import pytest


def test_lookup_kernel_registers_and_no_local_memory():
    if shutil.which('cuobjdump') is None:
        pytest.skip('cuobjdump unavailable')
    from gpt4roi_b200 import build, lib
    build.build()
    res = subprocess.run(['cuobjdump', '-res-usage', lib.LIB_PATH], capture_output=True, text=True)
    if res.returncode != 0:
        pytest.skip('cuobjdump unavailable')
    found = re.findall(r'Function (\S+):\s*\n\s*REG:(\d+) STACK:\d+ SHARED:\d+ LOCAL:(\d+)', res.stdout)
    usage = {n: (int(r), int(l)) for n, r, l in found if 'lookup_kernel' in n}
    assert len(usage) == 1, usage                     # no fp16 twin: integer only
    (name, (regs, local)), = usage.items()
    assert regs == 32 and local == 0, (name, regs, local)
    out = subprocess.run(['cuobjdump', '-sass', '-fun', name, lib.LIB_PATH], capture_output=True, text=True,
                         check=True).stdout
    assert not re.findall(r'\b(?:STL|LDL)(?:\.\w+)*\s', out)
