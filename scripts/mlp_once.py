"""One fused MLP forward at BASELINE config 3's shape (a short run for a profiler capture of mlp_fused_h3_kernel)."""
import sys
import torch
sys.path.insert(0, '.')
import cfm_b200
torch.manual_seed(0)
dev = torch.device('cuda:0')
m = cfm_b200.MLP(dim=784, w=256, time_varying=True).to(dev)
x = torch.randn(10000, 784, device=dev)
with torch.no_grad():
    for _ in range(4):
        y = m.vector_field(0.3, x)
torch.cuda.synchronize()
print(float(y.abs().max()))
