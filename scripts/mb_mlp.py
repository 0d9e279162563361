import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'comfyui-3d-pack_b200'))
import torch
from kiui.nn import MLP
dev = torch.device('cuda:0')
m = MLP(32, 1, 32, 2, bias=False).to(dev)
N = 20_000_000
x = torch.randn(N, 32, device=dev)
def tm(fn, n=3):
    fn(); torch.cuda.synchronize()
    a, b = torch.cuda.Event(True), torch.cuda.Event(True); a.record()
    for _ in range(n): fn()
    b.record(); torch.cuda.synchronize(); return a.elapsed_time(b) / n
with torch.no_grad():
    print('fused fwd ms', tm(lambda: m(x)))
    print('linear fwd ms', tm(lambda: torch.relu(x @ m.net[0].weight.T) @ m.net[1].weight.T))
xg = x.requires_grad_(True)
def fb():
    y = m(xg); y.sum().backward()
print('fused fwd+bwd ms', tm(fb))
def fb2():
    y = torch.relu(xg @ m.net[0].weight.T) @ m.net[1].weight.T; y.sum().backward()
print('linear fwd+bwd ms', tm(fb2))
