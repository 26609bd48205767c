"""Shadows the reference's data_loaders/motion_representation.py: everything the drivers import from it with
``from data_loaders.motion_representation import *`` keeps coming from the reference's own file (found further down
``sys.path``: cano_seq_smplx, get_repr_smplx, foot_detect, ...), except ``recover_from_repr_smpl`` (:332-398), which is routed
to the CUDA kernels whenever its inputs live on a CUDA device (test_amass_full.py:292, 406, 416-418, 428).
"""
import importlib.util
import os
import sys

from rohm_b200.motion_representation import recover_from_repr_smpl as _recover_b200

_here = os.path.abspath(os.path.dirname(__file__))
_ref = None
for _p in sys.path:
    _cand = os.path.join(os.path.abspath(_p or "."), "data_loaders", "motion_representation.py")
    if os.path.isfile(_cand) and os.path.dirname(_cand) != _here:
        _spec = importlib.util.spec_from_file_location("_rohm_reference_motion_representation", _cand)
        _ref = importlib.util.module_from_spec(_spec)
        _spec.loader.exec_module(_ref)
        break

if _ref is not None:
    globals().update({k: v for k, v in vars(_ref).items() if not k.startswith("__")})


def recover_from_repr_smpl(data_dict, recover_mode='joint_abs_traj', smplx_model=None, return_verts=False,
                           return_full_joints=False):
    first = next(iter(data_dict.values()))
    on_gpu = getattr(first, "is_cuda", False)
    if on_gpu and not return_full_joints:
        return _recover_b200(data_dict, recover_mode=recover_mode, smplx_model=smplx_model, return_verts=return_verts)
    if _ref is None:
        raise RuntimeError("recover_from_repr_smpl: CPU tensors / return_full_joints need the reference's "
                           "data_loaders/motion_representation.py on sys.path (rohm_b200 has no CPU path)")
    return _ref.recover_from_repr_smpl(data_dict, recover_mode=recover_mode, smplx_model=smplx_model,
                                       return_verts=return_verts, return_full_joints=return_full_joints)
