"""Generate tests/golden/eq_response.npz by running the UNMODIFIED reference on CPU.

    DASP_REFERENCE=/path/to/dasp-pytorch python tools/make_eq_response_golden.py

The EQ's sections are built with the reference's own ``signal.biquad`` calls, exactly as its ``parametric_eq`` builds
them (functional.py:211-265), and the response is the reference's ``signal.fft_sosfreqz(sos, n_fft)`` (signal.py:14-32)
in fp32 and in fp64, at two grid sizes.  Six items drawn over the ``ParametricEQ`` ranges at 44.1 kHz; item 0 has its
low shelf at 20 Hz, item 1 its low shelf at the minimum Q.  To keep the fixture small, only some bins of each grid are
stored (``bins_<n_fft>``): every bin up to a few hundred Hz, where the low shelves and their fp32 trouble sit, and an
even subsample of the rest up to sr/2.  Only this file is written: the fixtures of oracle/make_golden.py are left as
they are.
"""
import os
import sys

import numpy as np
import torch

if os.environ.get("DASP_REFERENCE"):
    sys.path.insert(0, os.environ["DASP_REFERENCE"])
import dasp_pytorch  # noqa: E402  (the reference)
import dasp_pytorch.signal as RS  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "eq_response.npz")
KINDS = ("low_shelf", "peaking", "peaking", "peaking", "peaking", "high_shelf")
NFFTS = (4096, 131072)
LOW_BINS = {4096: 64, 131072: 512}       # every bin below about 700 / 170 Hz
STRIDE = {4096: 16, 131072: 512}         # then every STRIDE-th bin, and sr/2


def kept_bins(n_fft):
    nb = n_fft // 2 + 1
    idx = set(range(LOW_BINS[n_fft])) | set(range(0, nb, STRIDE[n_fft])) | {nb - 1}
    return np.array(sorted(idx), dtype=np.int64)


def reference_sos(params, sr, dtype):
    """(bs, 6, 6) sections from the reference's signal.biquad, as its parametric_eq fills them"""
    p = [q.to(dtype).view(-1, 1, 1) for q in params]
    bs = p[0].shape[0]
    sos = torch.zeros(bs, 6, 6, dtype=dtype)
    for k, kind in enumerate(KINDS):
        b, a = RS.biquad(p[3 * k], p[3 * k + 1], p[3 * k + 2], sr, kind)
        sos[:, k, :] = torch.cat((b, a), dim=-1).view(bs, 6)
    return sos


def main():
    sr, bs = 44100, 6
    g = torch.Generator().manual_seed(66)
    p01 = torch.rand(bs, 18, generator=g)
    p01[0, 1] = 0.0          # low-shelf cut-off at 20 Hz
    p01[1, 2] = 0.0          # low-shelf Q at 0.1
    proc = dasp_pytorch.ParametricEQ(sr)
    d = proc.denormalize_param_dict(proc.extract_param_dict(p01))
    params = list(d.values())                                  # fp32, as the reference's Processor hands them on
    st = {"p01": p01.numpy(), "names": np.array(list(d.keys())), "sample_rate": np.array(sr),
          "params": torch.stack(params, 0).numpy(), "n_fft": np.array(NFFTS)}
    for n_fft in NFFTS:
        keep = kept_bins(n_fft)
        st[f"bins_{n_fft}"] = keep
        st[f"h32_{n_fft}"] = RS.fft_sosfreqz(reference_sos(params, sr, torch.float32), n_fft)[:, keep].numpy()
        st[f"h64_{n_fft}"] = RS.fft_sosfreqz(reference_sos(params, sr, torch.float64), n_fft)[:, keep].numpy()
    np.savez_compressed(OUT, **st)
    print(OUT, os.path.getsize(OUT) // 1024, "KiB")


if __name__ == "__main__":
    main()
