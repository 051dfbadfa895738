"""ps_mesh_render and ps_mesh_texture on test_pose's rendered scene: its six true depth maps at 1280 x 960 fused into a 512^3
volume over the scene's bounds (tools/mesh_bench.py's set-up) and meshed, then the mesh rendered into the six views and
textured at cell 8 from the six images.  Both calls run on device buffers through the C ABI, so no upload is timed.
Calls are timed with CUDA events (median, min and max over --reps calls after a warm-up), kernels by torch.profiler in a
separate run.  Prints (triangle, view) pairs per second, the covered pixels, the split between small and big triangles,
texels per second and the atlas bytes over the fill kernel's time against the 3.35 TB/s HBM bound of the H100 SXM data
sheet, with the card name and power limit read in the same run.

    python tools/render_bench.py [--reps N] [out.json]
"""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from popsift_b200 import api        # noqa: E402
from mesh_bench import _bounds, _time   # noqa: E402

KERNELS = ("rd_check_kernel", "rd_raster_kernel", "rd_big_kernel", "rd_resolve_kernel", "tx_select_kernel", "tx_fill_kernel")
HBM_TBPS = 3.35


def _profile(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    per = {}
    for e in prof.key_averages():
        for k in KERNELS:
            if k in e.key:
                per[k] = per.get(k, 0.0) + e.device_time_total / 1000.0
    return per


def main():
    import torch
    reps = 5
    args = sys.argv[1:]
    if "--reps" in args:
        i = args.index("--reps"); reps = int(args[i + 1]); del args[i:i + 2]
    out_path = args[0] if args else None
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    import test_depth as td
    imgs, cams, poses, truth = td._rendered(1.0)
    depths = [D.astype(np.float32) for D in truth]
    lo, hi = _bounds(depths, cams, poses)
    n = 512
    voxel = float((hi - lo).max() / (n - 9))
    vol = api.TsdfVolume(lo - 4 * voxel, voxel, (n, n, n))
    vol.integrate(imgs, cams, poses, depths, trunc=3 * voxel)
    mesh = vol.mesh()
    vol.free()
    lib = api.load_library()
    nv, nt = len(mesh.vertices), len(mesh.triangles)
    d_v = torch.from_numpy(mesh.vertices.view(np.float32).reshape(-1, 4).copy()).cuda()
    d_t = torch.from_numpy(mesh.triangles).cuda()
    h, w = imgs[0].shape
    V = len(imgs)
    dimg = [torch.from_numpy(im).cuda() for im in imgs]
    ddep = [torch.empty((h, w), dtype=torch.float32, device="cuda") for _ in range(V)]
    dtri = [torch.empty((h, w), dtype=torch.int32, device="cuda") for _ in range(V)]
    sizes = np.array([[w, h]] * V, np.int32)
    cam = api._c_cameras(cams)
    rig = api._c_rigids(poses)
    rrep = api.PsRenderReport()

    def render():
        rc = lib.ps_mesh_render(0, V, sizes.ctypes.data, cam.ctypes.data, rig, d_v.data_ptr(), nv, d_t.data_ptr(), nt,
                                C.byref(api.PsRenderParams(1e-3, 0)), (C.c_void_p * V)(*[d.data_ptr() for d in ddep]),
                                (C.c_void_p * V)(*[d.data_ptr() for d in dtri]), C.byref(rrep))
        assert rc == 0, api._last_error(lib)

    cell = 8
    cpr = api.atlas_cells_per_row(nt, cell)
    _, Wa, Ha = api.atlas_uv(0, cell, cpr)
    Ha = -(-nt // cpr) * cell
    d_atlas = torch.empty((Ha, Wa), dtype=torch.uint8, device="cuda")
    d_view = torch.empty(nt, dtype=torch.int32, device="cuda")
    c_img = (api.PsImage * V)(*[api.PsImage(d.data_ptr(), w, w, h) for d in dimg])
    trep = api.PsTextureReport()
    tprm = api.PsTextureParams(cell, cpr, 0.01, 0.1, 1e-3, 0)

    def texture():
        rc = lib.ps_mesh_texture(0, V, c_img, cam.ctypes.data, rig, (C.c_void_p * V)(*[d.data_ptr() for d in ddep]), d_v.data_ptr(), nv,
                                 d_t.data_ptr(), nt, C.byref(tprm), d_atlas.data_ptr(), d_view.data_ptr(), C.byref(trep))
        assert rc == 0, api._last_error(lib)

    t_render = _time(render, reps)
    t_texture = _time(texture, reps)
    per_render = _profile(render)
    per_texture = _profile(texture)
    raster = sum(per_render.get(k, 0.0) for k in ("rd_raster_kernel", "rd_big_kernel", "rd_resolve_kernel"))
    fill = per_texture.get("tx_fill_kernel", float("nan"))
    texels = Wa * Ha
    res = dict(gpu=q.stdout.strip(), volume=n, voxel=voxel, views=V, image=(w, h), triangles=nt, vertices=nv,
               render=dict(call_ms=t_render, kernels_ms=per_render, report=dict(drawn=rrep.n_drawn, big=rrep.n_big, covered=rrep.n_covered),
                           pairs=nt * V, pairs_per_s=nt * V / (t_render[0] / 1e3), small=rrep.n_drawn - rrep.n_big,
                           covered_share=rrep.n_covered / (V * w * h), raster_kernels_ms=raster),
               texture=dict(call_ms=t_texture, kernels_ms=per_texture, report=dict(viewed=trep.n_viewed, fallback=trep.n_fallback),
                            atlas=(Wa, Ha), texels=texels, texels_per_s=texels / (t_texture[0] / 1e3), fill_TBps=texels / (fill / 1e3) / 1e12,
                            fill_share_of_hbm=texels / (fill / 1e3) / 1e12 / HBM_TBPS))
    print(json.dumps(res, indent=1, default=str))
    if out_path:
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1, default=str)


if __name__ == "__main__":
    main()
