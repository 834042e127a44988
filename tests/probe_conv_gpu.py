"""GPU probe: every hot-path conv shape on both conv paths vs a torch fp64 reference."""
import sys, time
import torch
sys.path.insert(0, '.')
import diffusiondepth_b200 as dd

torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
dev = torch.device('cuda:0')
print(torch.cuda.get_device_name(0), torch.cuda.get_device_capability(0))
shapes = [(16, 64), (64, 256), (256, 256), (256, 64), (64, 16)]
sizes = [(2, 24, 40), (1, 8, 16), (1, 13, 21), (2, 64, 96)]
for simt in (True, False):
    eng = dd.DenoiseEngine('swin', 1, (8, 16), (4, 8), 2, dev, cuda_graph=False, simt_conv=simt)
    for (cin, cout) in shapes:
        for (B, H, W) in sizes:
            g = torch.Generator(device='cpu').manual_seed(cin * 1000 + cout + H)
            x = torch.randn(B, cin, H, W, generator=g).to(dev)
            w = (torch.randn(cout, cin, 3, 3, generator=g) * 0.05).to(dev)
            b = torch.randn(cout, generator=g).to(dev)
            try:
                y = eng.conv3x3(x, w, b)
                torch.cuda.synchronize()
            except Exception as e:
                print(f"simt={simt} {cin}->{cout} {B}x{H}x{W}: EXC {e}")
                raise
            ref = torch.nn.functional.conv2d(x.double(), w.double(), b.double(), padding=1)
            err = (y.double() - ref).abs().max().item()
            scale = ref.abs().max().item()
            ref32 = torch.nn.functional.conv2d(x, w, b, padding=1)
            err32 = (ref32.double() - ref).abs().max().item()
            print(f"simt={int(simt)} {cin:3d}->{cout:3d} {B}x{H}x{W}: max|err|={err:.3e} (rel {err/scale:.2e}); torch-fp32 err {err32:.3e}")
    eng.close()
# timing of the dominant shape
eng = dd.DenoiseEngine('swin', 1, (8, 16), (4, 8), 2, dev, cuda_graph=False)
x = torch.randn(4, 256, 176, 608, device=dev); w = torch.randn(256, 256, 3, 3, device=dev) * 0.02; b = torch.zeros(256, device=dev)
for _ in range(2):
    t = time.time(); y = eng.conv3x3(x, w, b); torch.cuda.synchronize(); print('conv3x3 full-size wall (incl. layout/split):', time.time() - t)
ref = torch.nn.functional.conv2d(x[:1, :, :32, :64].double(), w.double(), b.double(), padding=1)
print('full-size corner err', (y[:1, :, :31, :63].double() - ref[:, :, :31, :63]).abs().max().item())
