"""CPU guard on the machine code of the wgmma GEMM (csrc/gemm_wgmma.cu), read from the built library with cuobjdump.

Every `gemm_bf16_wgmma` instantiation, bf16 and fp16, must
  * keep its accumulators in registers: no local-memory traffic (STL / LDL);
  * close each k-block's MMAs with the commit of the same group: no empty `HGMMA.64x8x16 ... RZ` group, which ptxas
    emits when wgmma.commit_group sits in another basic block than the MMAs it closes -- `wait_group 1` then counts
    the empty group as the one left in flight and every k-block's MMAs finish before the next is issued."""
import re
import shutil
import subprocess

import pytest


@pytest.fixture(scope='module')
def gemm_sass():
    if shutil.which('cuobjdump') is None:
        pytest.skip('cuobjdump unavailable')
    from gpt4roi_b200 import build, lib
    build.build()
    res = subprocess.run(['cuobjdump', '-res-usage', lib.LIB_PATH], capture_output=True, text=True)
    if res.returncode != 0:
        pytest.skip('cuobjdump unavailable')
    names = sorted(set(re.findall(r'Function (\S*gemm_bf16_wgmma\S*):', res.stdout)))
    assert names, 'no gemm_bf16_wgmma kernel in %s' % lib.LIB_PATH
    out = subprocess.run(['cuobjdump', '-sass', '-fun', ','.join(names), lib.LIB_PATH],
                         capture_output=True, text=True, check=True).stdout
    funcs = {}
    for chunk in re.split(r'\n\s*Function : ', out)[1:]:
        name = chunk.split('\n', 1)[0].strip()
        funcs[name] = chunk
    assert set(funcs) == set(names), (sorted(funcs), names)
    return funcs


def test_gemm_kernels_cover_both_types(gemm_sass):
    assert any(n.startswith('_ZN3g4r15') for n in gemm_sass), 'bf16 GEMM kernels missing'
    assert any(n.startswith('_ZN5g4r_h15') for n in gemm_sass), 'fp16 GEMM kernels missing'


def test_gemm_kernels_do_not_spill(gemm_sass):
    bad = {n: len(re.findall(r'\b(?:STL|LDL)(?:\.\w+)*\s', s)) for n, s in gemm_sass.items()}
    assert not any(bad.values()), {n: c for n, c in bad.items() if c}


def test_gemm_mainloops_have_no_empty_commit_group(gemm_sass):
    bad = {n: len(re.findall(r'HGMMA\.64x8x16\.\S+\s+RZ', s)) for n, s in gemm_sass.items()}
    assert not any(bad.values()), {n: c for n, c in bad.items() if c}
    for n, s in gemm_sass.items():
        assert 'HGMMA.' in s and 'WARPGROUP.DEPBAR.LE gsb0, 0x1' in s, n
