"""fp64 restatement of convolution_reverberation with a true-stereo (four-channel) impulse response, for the tests.

The IR's channels are input-major: channel 2 i + o is the path from input channel i to output channel o (L->L, L->R,
R->L, R->R), so  wet_o = sum_i x_i * h[2 i + o]  (causal convolution cropped to n), y = (1 - mix) x + mix wet.  Written
as one 2 x 2 matrix of filters per item, independently of tests/conv_oracle.py, which it defers to for 1 or 2 channels;
tests/test_conv_reverb_ts_host.py ties the two together (a diagonal IR is the stereo IR, and a true-stereo IR is the
two stereo calls its rows make)."""
import math

import torch

import conv_oracle


def convolution_reverberation(x, sample_rate, ir, mix, method: str = "fft"):
    """x (bs, 1|2, n), ir (bs, 1|2|4, L), mix (bs elements) -> (bs, 2, n); mono x feeds both inputs"""
    if ir.shape[1] != 4:
        return conv_oracle.convolution_reverberation(x, sample_rate, ir, mix, method=method)
    bs, chs, n = x.shape
    if chs == 1:
        x = x.repeat(1, 2, 1)
    L = ir.shape[-1]
    h = ir.reshape(bs, 2, 2, L)                                  # [item, input i, output o, tap]
    if method == "direct":
        # one grouped conv1d per item: output channel o of item b sums input channels i with kernel h[b, i, o]
        w = torch.flip(h, dims=[-1]).transpose(1, 2).reshape(bs * 2, 2, L)
        xp = torch.nn.functional.pad(x, (L - 1, 0)).reshape(1, bs * 2, n + L - 1)
        wet = torch.nn.functional.conv1d(xp, w, groups=bs).reshape(bs, 2, n)
    else:
        m = 1 << math.ceil(math.log2(n + L - 1))
        wet = torch.fft.irfft(torch.einsum("bif,biof->bof", torch.fft.rfft(x, m), torch.fft.rfft(h, m)), m)[..., :n]
    mix = mix.reshape(bs, 1, 1)
    return (1.0 - mix) * x + mix * wet
