"""Training step of the 7B LLaMA stack (SURVEY.md 8(a) row 14, first slice; BASELINE config 4 shape: 336 px
prompt of 706 tokens, per-GPU batch 4 = global batch 32 on 8 GPUs): forward + backward + gradient all-reduce +
AdamW on the sm_90a kernels, synthetic inputs_embeds/labels, random-init weights.
  python tools/bench_train.py [--batch 4] [--steps 5] [--warmup 2]
  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P tools/bench_train.py
Prints one JSON line (rank 0).  The SPI / projector / embedding backward is not part of this slice."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gpt4roi_b200 import lib as L  # noqa: E402
from gpt4roi_b200.engine import EngineConfig, random_state_dicts  # noqa: E402
from gpt4roi_b200.train import LayerBucketAllReduce, LlamaTrainStack, train_step  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=4)
    ap.add_argument('--seq', type=int, default=706)
    ap.add_argument('--layers', type=int, default=32)
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--full', action='store_true', help='whole stage-2 step (BASELINE config 4): CLIP (frozen) + SPI + projector + '
                    'embeddings + LLaMA, 336 px, 8 RoIs/img, 128 text tokens; default is the LLaMA stack only')
    ap.add_argument('--ncu', action='store_true', help='one steady-state step inside a cudaProfiler window (run under '
                    'ncu --profile-from-start off)')
    a = ap.parse_args()
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(local)
    dev = 'cuda:%d' % local
    reducer = None
    if world > 1:
        import torch.distributed as dist
        if os.environ.get('NCCL_DEBUG', 'VERSION') in ('', 'VERSION'):
            os.environ['NCCL_DEBUG'] = 'WARN'
        dist.init_process_group('nccl', device_id=torch.device(dev))
        reducer = LayerBucketAllReduce()
    if a.full:
        return full_step(a, world, rank, dev, reducer)
    cfg = EngineConfig(image_size=336, vit_layers=0, n_layers=a.layers)
    sd, _ = random_state_dicts(cfg, dev, seed=0)                 # same weights on every rank (same seed)
    stack = LlamaTrainStack(cfg, sd, dev, lr=2e-5)
    del sd
    torch.cuda.empty_cache()
    g = torch.Generator(device='cpu').manual_seed(100 + rank)    # a different micro-batch per rank
    x = (torch.randn(a.batch, a.seq, cfg.hidden, generator=g) * 0.5).to(dev, torch.bfloat16)
    labels = torch.randint(0, cfg.vocab, (a.batch, a.seq), generator=g).to(dev)
    targets = torch.full_like(labels, -100)
    targets[:, :-1] = labels[:, 1:]
    losses = []
    for _ in range(a.warmup):
        loss, _ = train_step(stack, x, targets, reducer, world)
        losses.append(loss.item())
    if world > 1:
        torch.distributed.barrier()
    torch.cuda.synchronize()
    l0 = L.LAUNCHES
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        loss, _ = train_step(stack, x, targets, reducer, world)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.steps
    if world > 1:
        t = torch.tensor([ms], device=dev)
        torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.MAX)
        ms = t.item()
    losses.append(loss.item())
    if rank == 0:
        n_params = sum(f.numel() + 2 * cfg.hidden for f in stack.wflat) + stack.w_top['lm_head'].numel() + cfg.hidden
        tokens = a.batch * a.seq
        # 6 flop / parameter / token (fwd 2 + bwd 4) + causal attention (fwd 2*2*L*hid/2, bwd 2.5x incl. recompute)
        attn = a.layers * a.batch * (4.0 * a.seq * a.seq * cfg.hidden / 2) * 3.5
        flops = 6.0 * n_params * tokens + attn
        print(json.dumps(dict(metric='train_step_llama_stack_tokens_per_sec', value=world * tokens / (ms / 1e3), unit='tokens/s',
                              n_gpus=world, ms_per_step=ms, steps=a.steps, warmup=a.warmup,
                              config=dict(workload='7B LLaMA stack fwd+bwd+allreduce+AdamW, bf16, seq %d, per-GPU batch %d' % (a.seq, a.batch),
                                          layers=a.layers, params=n_params, global_batch=world * a.batch),
                              model_tflops_per_gpu=flops / (ms / 1e3) / 1e12, gpu_launches_per_step=(L.LAUNCHES - l0) // a.steps,
                              peak_mem_GB=torch.cuda.max_memory_allocated() / 1e9, losses=[round(v, 4) for v in losses],
                              scope='LLaMA decoder stack + lm_head + loss only (SPI/projector/embedding backward not built)')),
              flush=True)
    if world > 1:
        torch.distributed.destroy_process_group()


def full_step(a, world, rank, dev, reducer):
    from bench import synthetic_inputs
    from gpt4roi_b200.train import Stage2Trainer
    cfg = EngineConfig(image_size=336, n_layers=a.layers)
    sd, vit_sd = random_state_dicts(cfg, dev, seed=0)
    tr = Stage2Trainer(cfg, sd, vit_sd, dev, lr=2e-5, reducer=reducer, world_size=world,
                       shard_optimizer=os.environ.get('G4R_SHARD') == '1')   # G4R_DDP_SM_RESERVE / NCCL_MAX_CTAS / G4R_SHARD from the env
    del sd, vit_sd
    torch.cuda.empty_cache()
    ids, images, boxes = synthetic_inputs(cfg, a.batch, 8, 128, seed=100 + rank)   # a different micro-batch per rank
    ids, images = ids.to(dev), images.to(dev)
    labels = ids.clone()
    labels[:, : cfg.num_patches + 3] = -100
    labels[ids == cfg.bbox_token] = -100
    losses = []
    for _ in range(a.warmup):
        losses.append(tr.step(ids, images, boxes, labels).item())
    if a.ncu:
        torch.cuda.synchronize()
        torch.cuda.profiler.start()
        tr.step(ids, images, boxes, labels)
        torch.cuda.synchronize()
        torch.cuda.profiler.stop()
        return
    if world > 1:
        torch.distributed.barrier()
    torch.cuda.synchronize()
    l0 = L.LAUNCHES
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        loss = tr.step(ids, images, boxes, labels)
    tr.stack.sync_optimizer()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.steps
    if world > 1:
        t = torch.tensor([ms], device=dev)
        torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.MAX)
        ms = t.item()
    losses.append(loss.item())
    if rank == 0:
        n_params = sum(f.numel() + 2 * cfg.hidden for f in tr.stack.wflat) + tr.stack.w_top['lm_head'].numel() + cfg.hidden \
            + sum(v.numel() for v in tr.master.values())
        print(json.dumps(dict(metric='train_step_stage2_samples_per_sec', value=world * a.batch / (ms / 1e3), unit='samples/s',
                              n_gpus=world, ms_per_step=ms, steps=a.steps, warmup=a.warmup,
                              config=dict(workload='stage-2 step (ViT frozen), 7B, bf16, 336 px, 8 RoIs/img, 128 text tokens (L=%d), per-GPU batch %d'
                                          % (ids.shape[1], a.batch), layers=a.layers, trained_params=n_params, global_batch=world * a.batch),
                              tokens_per_sec=world * a.batch * ids.shape[1] / (ms / 1e3), gpu_launches_per_step=(L.LAUNCHES - l0) // a.steps,
                              peak_mem_GB=torch.cuda.max_memory_allocated() / 1e9, losses=[round(v, 4) for v in losses],
                              sm_reserve=tr.sm_reserve, nccl_max_ctas=os.environ.get('NCCL_MAX_CTAS'), sharded=tr.shard,
                              data='synthetic images / boxes / tokens, random-init weights')), flush=True)
    if world > 1:
        torch.distributed.destroy_process_group()


if __name__ == '__main__':
    main()
