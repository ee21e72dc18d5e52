import os, sys, ctypes as C
os.environ["BGS_TIMELINE"] = "1"; os.environ["BGS_TIMELINE_SORT"] = "1"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import bevy_gaussian_splatting_b200 as B
cloud = B.random_gaussians_3d_seeded(6_000_000, 0)
pl = B.GaussianSplattingPlugin(0); h = pl.add_cloud(cloud, f16=True)
s = B.CloudSettings(global_scale=0.02, rasterize_mode=B.RasterizeMode.Depth)   # Depth: projection waits, the sort runs alone
v = B.headless_view(1920, 1080)
for _ in range(5): pl.render_view(h, s, v, fmt="rgba8_srgb", to_host=False)
buf = np.zeros((4096, 8), np.uint64); g = C.c_uint32()
lib = pl._lib; lib.bgs_debug_timeline_.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32)]
lib.bgs_debug_timeline_(pl._ctx, buf.ctypes.data_as(C.c_void_p), C.byref(g))
nt = int((buf[:, 0] != 0).sum())
print("tiles stamped:", nt)
t = buf[:nt, :6].astype(np.int64); t = (t - t[:, :1]) / 1980.0   # clock64 cycles -> us at 1.98 GHz (H100 SXM max SM clock), per-tile origin
names = ["tile start", "ranked", "scanned", "smem scatter", "post-lookback", "written"]
for i, nm in enumerate(names):
    col = t[:, i]; print(f"{nm:14s} min {col.min():7.2f} median {np.median(col):7.2f} max {col.max():7.2f} us")
print("per-phase medians:", np.median(np.diff(t, axis=1), axis=0).round(2))
print("look-back duration by tile idx (every 16):", (t[::16, 4] - t[::16, 3]).round(2))
print(pl.stage_times_us())
