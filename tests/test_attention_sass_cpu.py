"""CPU guard on the machine code of the wgmma attention forward (csrc/attention_wgmma.cu), read from the built library
with cuobjdump: every `fa_fwd_wgmma` instantiation, bf16 and fp16, including the chunk-over-KV-cache mode
(g4r_attention_cached_*), keeps its S and O accumulators in registers -- no local-memory traffic (STL / LDL)."""
import re
import shutil
import subprocess

import pytest


def test_attention_kernels_do_not_spill():
    if shutil.which('cuobjdump') is None:
        pytest.skip('cuobjdump unavailable')
    from gpt4roi_b200 import build, lib
    build.build()
    res = subprocess.run(['cuobjdump', '-res-usage', lib.LIB_PATH], capture_output=True, text=True)
    if res.returncode != 0:
        pytest.skip('cuobjdump unavailable')
    names = sorted(set(re.findall(r'Function (\S*fa_fwd_wgmma\S*):', res.stdout)))
    # D in {64, 128}: non-causal, causal, and the cached mode (third template flag), each for bf16 and fp16
    assert len(names) == 12, names
    assert sum('ELb1ELb1E' in n for n in names) == 4, names
    out = subprocess.run(['cuobjdump', '-sass', '-fun', ','.join(names), lib.LIB_PATH],
                         capture_output=True, text=True, check=True).stdout
    funcs = {chunk.split('\n', 1)[0].strip(): chunk for chunk in re.split(r'\n\s*Function : ', out)[1:]}
    assert set(funcs) == set(names), (sorted(funcs), names)
    bad = {n: len(re.findall(r'\b(?:STL|LDL)(?:\.\w+)*\s', s)) for n, s in funcs.items()}
    assert not any(bad.values()), {n: c for n, c in bad.items() if c}
