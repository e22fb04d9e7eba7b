"""Sub-phase stamps of ONE epilogue chunk (SDB_DBG bit 6, sdb_debug_trace): epilogue warp 0, first chunk of the first
tile. Columns are SM clocks relative to accumulator-ready: accumulator load done, fused math done, staging stored + proxy
fence done, chunk finished (TMA store issued + statistics), whole epilogue finished (all chunks, stores read)."""
import ctypes as C, os, statistics, sys, torch
sys.path.insert(0, ".")
import sdb200
from sdb200 import ops
dev = torch.device("cuda:0")
lib = sdb200.lib.load()
M, N, K = 8192, 320, 960
g = torch.Generator().manual_seed(0)
a = torch.randn(M, K, generator=g).half().to(dev); b = (torch.randn(N, K, generator=g) * K ** -0.5).half().to(dev)
bias = torch.randn(N, generator=g).to(dev); res = torch.randn(M, N, generator=g).to(dev)
x4 = torch.randn(2, 64, 64, 320, generator=g).half().to(dev); w9 = (torch.randn(N, 9 * 320, generator=g) * 0.02).half().to(dev)
film = torch.randn(2, N, generator=g).to(dev)
ag = torch.randn(M, 320, generator=g).half().to(dev); wg = (torch.randn(2560, 320, generator=g) * 0.05).half().to(dev); bg = torch.randn(2560, generator=g).to(dev)
SLOT = 8 + 8 * 160
def run(name, fn):
    ops.RECORD = []
    fn()
    rec, ops.RECORD = ops.RECORD[0], None
    d = rec[0]
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for _ in range(5): lib.sdb_gemm(C.byref(d), st)
    torch.cuda.synchronize()
    ts = []
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda._sleep(2_000_000); e0.record()
        for _ in range(20): lib.sdb_gemm(C.byref(d), st)
        e1.record(); torch.cuda.synchronize(); ts.append(e0.elapsed_time(e1) / 20 * 1e3)
    buf = torch.zeros(SLOT * 4, dtype=torch.int64, device=dev)
    lib.sdb_debug_trace(C.c_void_p(buf.data_ptr()), buf.numel())
    for _ in range(3): lib.sdb_gemm(C.byref(d), st)
    lib.sdb_debug_trace(None, 0); torch.cuda.synchronize()
    r = buf.cpu().view(-1, SLOT)[2]; grid = int(r[0]); c = r[8:8 + 8 * min(grid, 160)].view(-1, 8)
    w = {k: int(c[:, k].median()) for k in range(2, 8)}
    t0 = w[6]
    print(f"{name:40s} {statistics.median(ts):7.2f} us | bn {int(r[1])} grid {grid} | accrdy {t0:6d} | ld {w[3]-t0:5d} math {w[4]-t0:5d} "
          f"staged {w[5]-t0:5d} chunk {w[2]-t0:5d} | epilogue {w[7]-t0:6d} clk")
print("SDB_DBG =", os.environ.get("SDB_DBG", "0"))
kw = dict(block_n=160, pair=1)
run("1x1 f32", lambda: ops.gemm(a, b, bias=bias, want_f32=True, **kw))
run("1x1 f32 + residual", lambda: ops.gemm(a, b, bias=bias, residual=res, want_f32=True, **kw))
run("1x1 f32 + stats", lambda: ops.gemm(a, b, bias=bias, want_f32=True, rows_per_sample=4096, want_stats=True, stats_group=10, **kw))
run("1x1 f16", lambda: ops.gemm(a, b, bias=bias, want_f16=True, **kw))
run("1x1 f16+lo + residual", lambda: ops.gemm(a, b, bias=bias, residual=res, want_lo=True, **kw))
run("3x3 f32 + film + stats", lambda: ops.gemm(x4, w9, taps=9, bias=bias, film=film, want_f32=True, want_stats=True, stats_group=10, **kw))
run("3x3 f32 + residual + stats", lambda: ops.gemm(x4, w9, taps=9, bias=bias, residual=res, want_f32=True, want_stats=True, stats_group=10, **kw))
run("geglu 8192x2560x320 bn256 pair", lambda: ops.gemm(ag, wg, bias=bg, act=ops.ACT_GEGLU, want_f16=True, block_n=256, pair=2))
run("geglu 8192x2560x320 bn256 single", lambda: ops.gemm(ag, wg, bias=bg, act=ops.ACT_GEGLU, want_f16=True, block_n=256, pair=1))
run("geglu 8192x2560x320 bn128 single", lambda: ops.gemm(ag, wg, bias=bg, act=ops.ACT_GEGLU, want_f16=True, block_n=128, pair=1))
