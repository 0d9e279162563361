import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'comfyui-3d-pack_b200'))
import torch
from kiui.gridencoder import GridEncoder
dev = torch.device('cuda:0')
enc = GridEncoder(num_levels=16).to(dev)
N = 20_000_000
# samples along rays through the r=0.5 ball (correlated like real marching)
o = torch.randn(N // 200, 3, device=dev); o = o / o.norm(dim=1, keepdim=True) * 1.75
d = -o / 1.75 + 0.2 * torch.randn_like(o); d = d / d.norm(dim=1, keepdim=True)
t = torch.linspace(1.25, 2.25, 200, device=dev)
x = (o[:, None, :] + d[:, None, :] * t[None, :, None]).reshape(-1, 3).clamp(-1, 1).contiguous()
g = torch.rand(N, 32, device=dev)
def tm(fn, n=3):
    fn(); torch.cuda.synchronize()
    a, b = torch.cuda.Event(True), torch.cuda.Event(True); a.record()
    for _ in range(n): fn()
    b.record(); torch.cuda.synchronize(); return a.elapsed_time(b) / n
out = enc(x)
print('fwd ms', tm(lambda: enc(x)))
def bw():
    enc.embeddings.grad = None
    out = enc(x); out.backward(g)
print('fwd+bwd ms', tm(bw))
xr = torch.rand(N, 3, device=dev) * 2 - 1
print('fwd random ms', tm(lambda: enc(xr)))
def bw2():
    enc.embeddings.grad = None
    out = enc(xr); out.backward(g)
print('fwd+bwd random ms', tm(bw2))
