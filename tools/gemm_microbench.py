import ctypes as C, os, sys, json
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
import torch
import dwbc_b200
from dwbc_b200 import _lib as L
lib = L.lib()
lib.dwbc_debug_gemm.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
M, N, K = 40960, 128, 128
nbuf = 8
X = [torch.randn(M, K, device="cuda") for _ in range(nbuf)]; Y = [torch.empty(M, N, device="cuda") for _ in range(nbuf)]
W = torch.randn(N, K, device="cuda"); b = torch.randn(N, device="cuda"); dW = torch.zeros(N, K, device="cuda"); db = torch.zeros(N, device="cuda")
def run(mode, tc, i):
    if mode == 0: return lib.dwbc_debug_gemm(0, tc, X[i].data_ptr(), K, W.data_ptr(), K, Y[i].data_ptr(), N, b.data_ptr(), None, M, N, K, 1, L.stream_ptr())
    if mode == 1: return lib.dwbc_debug_gemm(1, tc, X[i].data_ptr(), K, W.data_ptr(), N, Y[i].data_ptr(), N, None, None, M, N, K, 0, L.stream_ptr())
    return lib.dwbc_debug_gemm(2, tc, X[i].data_ptr(), N, Y[i].data_ptr(), K, dW.data_ptr(), K, None, db.data_ptr(), N, K, M, 0, L.stream_ptr())
out = {}
for mode in (0, 1, 2):
    for tc in (0, 1):
        for i in range(nbuf): run(mode, tc, i)
        torch.cuda.synchronize(); torch.cuda._sleep(20_000_000)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for r in range(3):
            for i in range(nbuf): run(mode, tc, i)
        e1.record(); torch.cuda.synchronize()
        out[f"mode{mode}_tc{tc}"] = round(e0.elapsed_time(e1) * 1e3 / (3 * nbuf), 2)
print(json.dumps(dict(us=out)))
if len(sys.argv) > 1 and sys.argv[1] == "stamps":
    buf = torch.zeros(148 * 64, dtype=torch.int64, device="cuda")
    lib.dwbc_debug_set_tc_cycle_buffer.argtypes = [C.c_void_p]
    lib.dwbc_debug_set_tc_cycle_buffer(buf.data_ptr())
    run(int(sys.argv[2]) if len(sys.argv) > 2 else 0, 1, 0); torch.cuda.synchronize()
    c = buf.view(148, 64).cpu()
    for b in (0, 1, 147):
        row = c[b]; t0 = int(row[0])
        print("CTA", b, {k: int(row[k]) - t0 for k in range(64) if int(row[k]) > 0})
    lib.dwbc_debug_set_tc_cycle_buffer(None)
