"""CPU guard on the machine code of the per-request selection and stop kernels (ContinuousBatcher(request_options=True)),
read from the built library with cuobjdump: sample_tokens_rows_kernel<true> (g4r_sample_tokens_rows_proc_*, bf16 and
fp16) and stop_step_rows_kernel use no local memory, and templating the per-row kernel left the kernels beside it as they
were -- sample_tokens_rows_kernel<false> at 31 / 30 registers (bf16 / fp16) and the batch instances
sample_tokens_kernel<false|true>, sample_tokens_out_kernel<false|true> at 28 / 40 / 32 / 40."""
import re

from tests.test_rows_kernels_sass_cpu import _usage

BATCH = {'20sample_tokens_kernelILb0E': 28, '20sample_tokens_kernelILb1E': 40, '24sample_tokens_out_kernelILb0E': 32,
         '24sample_tokens_out_kernelILb1E': 40}


def test_new_kernels_use_no_local_memory():
    usage, _ = _usage()
    names = sorted(n for n in usage if '25sample_tokens_rows_kernelILb1E' in n or 'stop_step_rows_kernel' in n)
    assert len(names) == 3, names        # the processed rows kernel in bf16 and fp16, the stop lookup once
    assert not any(usage[n][1] for n in names), {n: usage[n] for n in names}


def test_existing_selection_kernels_keep_their_register_counts():
    usage, _ = _usage()
    rows = sorted(n for n in usage if '25sample_tokens_rows_kernelILb0E' in n)
    assert len(rows) == 2, rows
    for n in rows:
        assert usage[n] == ((30 if re.search(r'g4r_h', n) else 31), 0), (n, usage[n])
    for frag, regs in BATCH.items():
        hits = [n for n in usage if frag in n]
        assert len(hits) == 2, (frag, hits)
        for n in hits:
            assert usage[n] == (regs, 0), (n, usage[n], regs)
