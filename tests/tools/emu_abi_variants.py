"""rgbl_frame_rgbl_batch (extraction + LiDAR depth of a 2-frame batch) through the real C ABI of the EMULATED library
(tests/cuda_emu/build.py), compared bit for bit with the oracle, without a GPU:
    python tests/tools/emu_abi_variants.py
"""
import sys, os
ROOT = __import__('pathlib').Path(__file__).resolve().parent.parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / 'tests'))
from orb_slam3_rgbl_b200 import _lib
from cuda_emu import build
_lib.LIB_PATH = build.build_full()
import numpy as np, oracle
from orb_slam3_rgbl_b200 import frontend as F, synthetic as S
W,H=420,260
img=S.make_image(5,W,H); pts=S.make_pointcloud(5,n_azimuth=500)
P=S.lidar_projection_matrix().copy(); P[0,:]*=W/S.KITTI_W; P[1,:]*=H/S.KITTI_H
ctx=F.Context(W,H,600,max_batch=2,max_points=pts.shape[1])
res=F.frame_rgbl_batch(ctx,[img,img[:, ::-1].copy()],[pts,pts],P,F.make_depth_params(bf=S.KITTI_BF))
ctx.close()
for (k,d,dep,ur),im in zip(res,[img,img[:, ::-1].copy()]):
    rk,rd,_=oracle.Extractor(600)(im)
    rdep,rur,_,_=oracle.depth_from_pcd(pts,P,W,H,S.structuring_element("diamond",5),S.KITTI_BF,rk,rk)
    ok = len(k)==len(rk) and all((k[f]==rk[f]).all() for f in k.dtype.names) and (d==rd).all() and (dep==rdep).all() and (ur==rur).all()
    print("frame ok" if ok else "MISMATCH", len(k), int((dep>0).sum()))
