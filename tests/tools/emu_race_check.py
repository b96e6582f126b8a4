"""Race check of the emulated kernels (tests/cuda_emu) under ThreadSanitizer: every conflicting pair of accesses that is not
separated by a barrier / warp rendezvous is reported, whatever the timing.  Usage:
    bash tests/tools/emu_race_check.sh
(builds the emulated library with -fsanitize=thread and runs this file under LD_PRELOAD=libtsan for: the extraction pipeline and the
dilation kernel)."""
import ctypes as C, os, sys, numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import oracle
from cuda_emu import build
from orb_slam3_rgbl_b200 import _lib as L, synthetic as S
lib=C.CDLL(str(build.build_full(sanitize='thread')))
which=sys.argv[1]
if which=='extract':
    w,h=200,160; img=S.make_image(81,w,h); prm=L.OrbParams(200,1.2,3,12,7)
    ok,od,_=oracle.Extractor(200,1.2,3,12,7)(img)
    lib.emu_extract.argtypes=[C.c_void_p,C.c_void_p,C.c_int,C.c_int,C.c_int,C.c_void_p,C.c_void_p,C.c_int]
    kps=np.empty(1024,oracle.KP_DTYPE); desc=np.empty((1024,32),np.uint8)
    n=lib.emu_extract(C.byref(prm),L.ptr(img),w,h,img.strides[0],L.ptr(kps),L.ptr(desc),1024); print('extract',n,len(ok),(desc[:n]==od).all())
if which=='dilate':
    W,H=160,90; P=S.lidar_projection_matrix().astype(np.float32); pts=S.make_pointcloud(3,n_azimuth=300)
    P2=P.copy(); P2[0,:]*=W/S.KITTI_W; P2[1,:]*=H/S.KITTI_H
    lib.emu_depth_dilate.argtypes=[C.c_void_p,C.c_int,C.c_void_p,C.c_int,C.c_int,C.c_void_p,C.c_int,C.c_int,C.c_float,C.c_float,C.c_float,C.c_void_p,C.c_void_p]
    m=np.ascontiguousarray(S.structuring_element("diamond",5),np.uint8); p=np.ascontiguousarray(pts,np.float32)
    raw=np.empty((H,W),np.float32); out=np.empty((H,W),np.float32)
    lib.emu_depth_dilate(L.ptr(p),p.shape[1],L.ptr(np.ascontiguousarray(P2.reshape(12))),W,H,L.ptr(m),5,5,5.0,200.0,1.0,L.ptr(raw),L.ptr(out)); print('dilate done',(out>0).sum())
