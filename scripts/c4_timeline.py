"""Phase timeline of one iteration (it = 50) of the seeded float64-potential Sinkhorn solver at BASELINE config 4
(CFM_SK_TL=1): globaltimer marks of the first and the last CTA."""
import os, sys, torch, numpy as np
os.environ["CFM_SK_TL"] = "1"
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
names = ["iter start", "v staged", "dv_min read", "row phase done", "barrier", "sweep done", "barrier", "du verified", "combine done", "barrier (iter end)"]
t0 = int(marks[:, 0].min())
for c, tag in ((0, "CTA 0"), (1, "last CTA")):
    print(tag, ", ".join(f"{n} {(int(marks[c, i]) - t0) / 1e3:.1f}" for i, n in enumerate(names) if marks[c, i] > 0), "(us)")
