import os, sys, torch, numpy as np
os.environ["CFM_SK_TL"] = "2"
sys.path.insert(0, '.')
import cfm_b200
dev = torch.device('cuda:0')
g = torch.Generator().manual_seed(40)
x0, x1 = torch.randn(4096, 512, generator=g).to(dev), torch.randn(4096, 512, generator=g).to(dev)
sb = cfm_b200.OTPlanSampler("sinkhorn", reg=0.1, num_iter_max=100, stop_thr=0.0, warn=False)
for _ in range(3):
    sb.sample_plan(x0, x1)
torch.cuda.synchronize()
B = next(iter(sb._bufs.values()))
# the timeline marks open the Sinkhorn workspace: 16 per CTA, CTA 0 then the last CTA
marks = np.frombuffer(B["ws_sk"][:256].cpu().numpy().tobytes(), dtype=np.uint64).reshape(2, 16)
for c, tag in ((0, "CTA 0"), (1, "last CTA")):
    for off, who in ((0, "thread 0"), (5, "thread 511")):
        t0 = int(marks[c, 0 + off])
        print(tag, who, "chunk 1 (last iteration):", ", ".join(f"{n} {(int(marks[c, i + off]) - t0) / 1e3:.2f}" for i, n in enumerate(["start", "rows screened", "sync", "row LSE + sync", "columns screened"])), "us")
