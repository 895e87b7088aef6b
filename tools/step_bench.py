"""Quick full-step timing of the Trainer (not the contract bench; see bench.py). usage: step_bench.py [B] [ch] [gan]"""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "vqgan-training_b200"))
os.environ.setdefault("VQB_OFFLINE", "1")
import warnings

warnings.simplefilter("ignore")
import torch

import native
import vae_trainer as vt

RANK, WORLD = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
if WORLD > 1:  # torchrun: one process per GPU, NCCL
    import torch.distributed as dist
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
    dist.init_process_group("nccl")
    if RANK != 0:
        sys.stdout = open(os.devnull, "w")
B = int(sys.argv[1]) if len(sys.argv) > 1 else 8
ch = int(sys.argv[2]) if len(sys.argv) > 2 else 128
gan = len(sys.argv) > 3 and sys.argv[3] == "gan"
R = 256
tr = vt.Trainer("cuda", vae_ch=ch, do_clamp=True, do_ganloss=gan, disc_type="hinge", use_lecam=gan)
loader = iter(vt.SyntheticLoader(B, R))
torch.cuda.synchronize()
for i in range(3):
    t0 = time.time()
    out = tr.step(next(loader)[0])
    torch.cuda.synchronize()
    print(f"warmup {i}: {1e3 * (time.time() - t0):.1f} ms loss {float(out['overall_vae_loss']):.4f}", flush=True)
l0 = native.launch_count()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
K = 5
t0 = time.time()
e0.record()
for i in range(K):
    out = tr.step(next(loader)[0])
e1.record()
host_ms = 1e3 * (time.time() - t0) / K
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / K
tf = (3.107 if gan else 2.780) * B / (ms / 1e3) / 1e3
print(f"STEP B={B} ch={ch} gan={gan}: {ms:.2f} ms/step (host issue {host_ms:.2f} ms) = {B / ms * 1e3:.1f} img/s "
      f"~{tf:.3f} PFLOP/s nominal; launches/step {(native.launch_count() - l0) / K:.0f}; "
      f"loss {float(out['overall_vae_loss']):.4f}; max mem {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB", flush=True)
if os.environ.get("VQB_PROFILE", "0") == "1":
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        tr.step(next(loader)[0])
        torch.cuda.synchronize()
    print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=int(os.environ.get("VQB_PROFILE_ROWS", "40")),
                                    max_name_column_width=70))

    from torch.autograd import DeviceType
    evs = [e for e in prof.events() if e.device_type == DeviceType.CUDA]
    evs.sort(key=lambda e: e.time_range.start)
    if evs:
        span = (max(e.time_range.end for e in evs) - evs[0].time_range.start) / 1e3
        busy, gaps, cur_end = 0.0, [], evs[0].time_range.start
        for e in evs:
            s0, s1 = e.time_range.start, e.time_range.end
            if s0 > cur_end:
                gaps.append((s0 - cur_end, e.name))
                cur_end = s0
            if s1 > cur_end:
                busy += s1 - cur_end
                cur_end = s1
        print(f"GPU span {span:.2f} ms, busy {busy / 1e3:.2f} ms, idle {span - busy / 1e3:.2f} ms in {len(gaps)} gaps; "
              f"gaps > 5us: {sum(1 for g in gaps if g[0] > 5)} totalling {sum(g[0] for g in gaps if g[0] > 5) / 1e3:.2f} ms")
        from collections import Counter
        c = Counter()
        for g, name in gaps:
            if g > 5:
                c[name[:60]] += g
        for name, g in c.most_common(15):
            print(f"   idle before {name}: {g / 1e3:.2f} ms")

if WORLD > 1:
    torch.cuda.synchronize()
    dist.barrier()
    dist.destroy_process_group()
