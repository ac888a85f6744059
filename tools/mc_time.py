import os, sys, time, ctypes
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import torch, numpy as np
from nphm_b200 import _native
from conftest import sphere_volume
dev=torch.device('cuda:0')
vol=torch.from_numpy(sphere_volume(256,0.37)).to(dev)
L=_native.lib()
for it in range(6):
    torch.cuda.synchronize(); t0=time.perf_counter()
    p=_native.McParams(256,256,256,0,0,0,0.0)
    wsb=L.nphm_mc_workspace_bytes(ctypes.byref(p))
    ws=torch.empty(wsb,device=dev,dtype=torch.uint8)
    torch.cuda.synchronize(); t1=time.perf_counter()
    nv,nt=ctypes.c_longlong(0),ctypes.c_longlong(0)
    _native.check(L.nphm_mc_count(vol.data_ptr(),ctypes.byref(p),ws.data_ptr(),ctypes.byref(nv),ctypes.byref(nt),None))
    t2=time.perf_counter()
    verts=torch.empty(nv.value,3,device=dev,dtype=torch.float64); tris=torch.empty(nt.value,3,device=dev,dtype=torch.int64)
    torch.cuda.synchronize(); t3=time.perf_counter()
    _native.check(L.nphm_mc_emit(vol.data_ptr(),ctypes.byref(p),ws.data_ptr(),0,verts.data_ptr(),tris.data_ptr(),None))
    torch.cuda.synchronize(); t4=time.perf_counter()
    print('alloc ws %.3f ms  count %.3f ms  alloc out %.3f ms  emit %.3f ms  (nv %d nt %d)'%((t1-t0)*1e3,(t2-t1)*1e3,(t3-t2)*1e3,(t4-t3)*1e3,nv.value,nt.value))
