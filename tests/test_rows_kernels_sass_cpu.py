"""CPU guard on the machine code of the cache-row-table kernels (continuous batching with prefix reuse), read from the
built library with cuobjdump: fa_cached_rows_wgmma (g4r_attention_cached_rows_*) and kv_append_rows_at
(g4r_kv_append_rows_at_*), bf16 and fp16, use no local memory, and adding them left the kernels they sit beside as
they were -- the chunk attention's cached mode at 165 / 122 registers (D = 128 / 64, DESIGN.md section 3), the
attention's other modes and kv_append at their counts."""
import re
import shutil
import subprocess

import pytest

# register counts of the existing kernels (sm_90a, CUDA 12.9): (name fragment, template args) -> registers
EXISTING = {('fa_fwd_wgmma', 'ILi128ELb1ELb1E'): 165, ('fa_fwd_wgmma', 'ILi64ELb1ELb1E'): 122,
            ('fa_fwd_wgmma', 'ILi128ELb1ELb0E'): 168, ('fa_fwd_wgmma', 'ILi64ELb1ELb0E'): 119,
            ('fa_fwd_wgmma', 'ILi128ELb0ELb0E'): 142, ('fa_fwd_wgmma', 'ILi64ELb0ELb0E'): 102,
            ('kv_append_bf16', 'EPK'): 30}


def _usage():
    if shutil.which('cuobjdump') is None:
        pytest.skip('cuobjdump unavailable')
    from gpt4roi_b200 import build, lib
    build.build()
    res = subprocess.run(['cuobjdump', '-res-usage', lib.LIB_PATH], capture_output=True, text=True)
    if res.returncode != 0:
        pytest.skip('cuobjdump unavailable')
    found = re.findall(r'Function (\S+):\s*\n\s*REG:(\d+) STACK:\d+ SHARED:\d+ LOCAL:(\d+)', res.stdout)
    return {n: (int(r), int(l)) for n, r, l in found}, lib


def test_row_table_kernels_do_not_spill():
    usage, lib = _usage()
    names = sorted(n for n in usage if 'fa_cached_rows_wgmma' in n or 'kv_append_rows_at' in n)
    assert len(names) == 6, names      # attention D in {64, 128} and the append, each bf16 and fp16
    assert not any(usage[n][1] for n in names), {n: usage[n] for n in names}
    out = subprocess.run(['cuobjdump', '-sass', '-fun', ','.join(names), lib.LIB_PATH],
                         capture_output=True, text=True, check=True).stdout
    funcs = {chunk.split('\n', 1)[0].strip(): chunk for chunk in re.split(r'\n\s*Function : ', out)[1:]}
    assert set(funcs) == set(names), (sorted(funcs), names)
    bad = {n: len(re.findall(r'\b(?:STL|LDL)(?:\.\w+)*\s', s)) for n, s in funcs.items()}
    assert not any(bad.values()), {n: c for n, c in bad.items() if c}
    # the row-table attention runs the cached mode's body: the same register budget
    for n in names:
        if 'fa_cached_rows_wgmma' in n:
            assert usage[n][0] == (165 if 'ILi128E' in n else 122), (n, usage[n])


def test_existing_kernels_keep_their_register_counts():
    usage, _ = _usage()
    for (frag, args), regs in EXISTING.items():
        hits = [n for n in usage if re.search(r'\d%s%s' % (frag, args), n)]
        assert len(hits) == 2, (frag, args, hits)          # bf16 and fp16
        for n in hits:
            assert usage[n] == (regs, 0), (n, usage[n], regs)
