"""Launch each GEMM engine once or twice at the C2 layer size; `time [name]`: CUDA-event time per call."""
import ctypes
import sys

import torch

sys.path.insert(0, ".")
from neuraludf_b200 import _lib as L

lib = L.lib()
dev = torch.device("cuda")
P = 65536
X = torch.randn(P, 256, device=dev) * 0.1
W = torch.randn(256, 256, device=dev) * 0.06
b = torch.zeros(256, device=dev)
Y = torch.empty(P, 256, device=dev)
dW = torch.zeros(256, 256, device=dev)
st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
imgs = {}
for npl in (2, 3):
    im = torch.zeros(lib.nudf_tc_image_elems(256, 256, npl), dtype=torch.int16, device=dev)
    lib.nudf_tc_prepare_weights(L.ptr(W), 256, 256, 256, 0, npl, L.ptr(im), st)
    imgs[npl] = im

if len(sys.argv) > 1 and sys.argv[1] == "time":
    flush = torch.empty(64 * 1024 * 1024, device=dev)
    calls = {
        "wgrad_tc_fp32_operands": lambda: lib.nudf_wgrad(L.ptr(Y), 256, L.ptr(X), 256, 256, 256, P, L.ptr(dW), 256, 1, st),
        "dense_fp32_ffma2": lambda: lib.nudf_dense_forward(L.ptr(X), 256, L.ptr(W), 256, L.ptr(b), L.ptr(Y), 256, P, 256, 256, 2, st),
        "wgrad_fp32_ffma2": lambda: lib.nudf_wgrad(L.ptr(Y), 256, L.ptr(X), 256, 256, 256, P, L.ptr(dW), 256, 0, st),
        "dense_tc_fp32_operand": lambda: lib.nudf_dense_forward_tc(L.ptr(X), 256, L.ptr(imgs[2]), 2, L.ptr(b), L.ptr(Y), 256, P, 256, 256, 2, st),
    }
    for name, call in calls.items():
        if len(sys.argv) > 2 and name != sys.argv[2]:
            continue
        for _ in range(3):
            call()
        t = 0.0
        for _ in range(10):
            flush.zero_()
            a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); call(); e.record(); torch.cuda.synchronize()
            t += a.elapsed_time(e)
        print("%s: %.1f us" % (name, t / 10 * 1e3))
    sys.exit(0)
for _ in range(2):
    lib.nudf_dense_forward(L.ptr(X), 256, L.ptr(W), 256, L.ptr(b), L.ptr(Y), 256, P, 256, 256, 2, st)
    lib.nudf_dense_forward_tc(L.ptr(X), 256, L.ptr(imgs[2]), 2, L.ptr(b), L.ptr(Y), 256, P, 256, 256, 2, st)
    lib.nudf_dense_forward_tc(L.ptr(X), 256, L.ptr(imgs[3]), 3, L.ptr(b), L.ptr(Y), 256, P, 256, 256, 2, st)
    lib.nudf_wgrad(L.ptr(Y), 256, L.ptr(X), 256, 256, 256, P, L.ptr(dW), 256, 1, st)
    lib.nudf_wgrad(L.ptr(Y), 256, L.ptr(X), 256, 256, 256, P, L.ptr(dW), 256, 0, st)
torch.cuda.synchronize()
print("done")
