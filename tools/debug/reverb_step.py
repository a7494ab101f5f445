"""Two forward+backward iterations of the device-noise reverb at BASELINE config-4 geometry (one 128-item chunk),
for ncu captures: --launch-skip 17 -c 17 with the reverb kernel regex profiles the second iteration."""
import sys
import torch
sys.path.insert(0, ".")
import dasp_pytorch_b200 as D

dev = torch.device("cuda:0")
bs, n, L = int(sys.argv[1]) if len(sys.argv) > 1 else 132, 48000, 96000
x = torch.rand(bs, 2, n, device=dev, requires_grad=True)
p = [torch.rand(bs, device=dev, requires_grad=True) for _ in range(25)]
for _ in range(2):
    y = D.noise_shaped_reverberation(x, 44100, *p, num_samples=L, num_bandpass_taps=1023)
    y.square().mean().backward()
torch.cuda.synchronize()
