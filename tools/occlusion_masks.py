"""Writes the PROX joint occlusion masks, mask_joint/<recording>/mask_joint.npy, on the device: the job of the
reference's utils/get_occlusion_mask.py for any number of recordings, with one scene depth map per scene and every frame
of each recording (the reference script stops after 100).  Needs no pyrender, trimesh or smplx.

    python tools/occlusion_masks.py --prox_root PROX --body_model_path data/body_models/smplx_model \
        --init_body_path data/init_motions/init_prox_rgbd --save_mask_path mask_joint_prox \
        --recordings N0Sofa_00034_01 MPH1Library_00034_01

Reads scenes/<scene>.ply (the scene is the recording name up to its first '_'), cam2world/<scene>.json,
calibration/Color.json, the frames of recordings/<recording>/Color and each frame's fit
<init_body_path>/<recording>/results/<frame>/000.pkl (camera frame)."""
import argparse
import json
import os
import pickle
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from rohm_b200 import occlusion  # noqa: E402
from rohm_b200.body_model import BodyModel, load_faces  # noqa: E402


def read_fits(folder, frames):
    rows = {k: [] for k, _ in occlusion.PARAMS}
    for fr in frames:
        with open(os.path.join(folder, 'results', fr, '000.pkl'), 'rb') as f:
            d = pickle.load(f)
        for k, w in occlusion.PARAMS:
            rows[k].append(np.asarray(d[k], np.float32).reshape(w))
    return {k: np.stack(v) if v else np.zeros((0, w), np.float32) for (k, w), v in zip(occlusion.PARAMS, rows.values())}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--prox_root", required=True)
    ap.add_argument("--body_model_path", required=True)
    ap.add_argument("--init_body_path", required=True)
    ap.add_argument("--save_mask_path", required=True)
    ap.add_argument("--recordings", nargs="+", required=True)
    ap.add_argument("--device", default="cuda:0")
    args = ap.parse_args(argv)
    dev = torch.device(args.device)
    model = BodyModel.create(args.body_model_path, device=dev)
    faces = load_faces(args.body_model_path)
    with open(os.path.join(args.prox_root, 'calibration', 'Color.json')) as f:
        color = json.load(f)
    scenes, maps, map_of, lengths, params = [], [], [], [], []
    for rec in args.recordings:
        scene = rec.split('_')[0]
        if scene not in scenes:
            V, F = occlusion.read_ply(os.path.join(args.prox_root, 'scenes', scene + '.ply'))
            with open(os.path.join(args.prox_root, 'cam2world', scene + '.json')) as f:
                c2w = np.array(json.load(f))
            maps.append(occlusion.scene_depth(V.astype(np.float32), F, c2w))
            scenes.append(scene)
        map_of.append(scenes.index(scene))
        frames = occlusion.color_frames(os.listdir(os.path.join(args.prox_root, 'recordings', rec, 'Color')))
        params.append(read_fits(os.path.join(args.init_body_path, rec), frames))
        lengths.append(len(frames))
    p = {k: torch.from_numpy(np.concatenate([q[k] for q in params])).to(dev) for k, _ in occlusion.PARAMS}
    R = len(args.recordings)
    K = np.repeat(np.asarray(color['camera_mtx'], np.float64)[None], R, 0)
    k = np.repeat(np.asarray(color['k'], np.float64).reshape(1, -1), R, 0)
    mask = occlusion.joint_mask(model, faces, p, lengths, torch.stack(maps), map_of, K, k).cpu().numpy()
    off = np.concatenate([[0], np.cumsum(lengths)])
    for r, rec in enumerate(args.recordings):
        out = os.path.join(args.save_mask_path, rec)
        os.makedirs(out, exist_ok=True)
        np.save(os.path.join(out, 'mask_joint.npy'), mask[off[r]:off[r + 1]].astype(np.float64))
        print(f"{rec}: {lengths[r]} frames, {int((mask[off[r]:off[r + 1]] == 0).sum())} occluded joints")


if __name__ == "__main__":
    main()
