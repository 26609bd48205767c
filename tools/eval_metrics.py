"""Prints the metrics of the reference's eval_amass_full.py or eval_prox_egobody.py from the pickles its test scripts
write (or pipeline.result_dict / video_result_dicts), computed on the device by rohm_b200.metrics, with the scripts'
names and units.  Needs no reference checkout and none of the rendering packages the scripts import.

    python tools/eval_metrics.py amass --saved_data_path results.pkl --mask_scheme lower [--traj_mask_ratio 0.1]
    python tools/eval_metrics.py video --dataset egobody --saved_data_dir DIR --recordings rec_a rec_b \
        --floor_height -1.66 -0.81            (or --floor_json floors.json: {"rec_a": -1.66, ...})

For video, DIR/<recording>.pkl is read for every recording in the order given; each recording's floor height is the
one its scene has in the reference's tables."""
import argparse
import json
import os
import pickle
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from rohm_b200 import metrics  # noqa: E402


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    sub = ap.add_subparsers(dest="mode", required=True)
    a = sub.add_parser("amass")
    a.add_argument("--saved_data_path", required=True)
    a.add_argument("--mask_scheme", default="lower", choices=metrics.MASK_SCHEMES)
    a.add_argument("--traj_mask_ratio", default=0.0, type=float)
    v = sub.add_parser("video")
    v.add_argument("--dataset", required=True, choices=metrics.DATASETS)
    v.add_argument("--saved_data_dir", required=True)
    v.add_argument("--recordings", nargs="+", required=True)
    fl = v.add_mutually_exclusive_group(required=True)
    fl.add_argument("--floor_height", nargs="+", type=float)
    fl.add_argument("--floor_json", help="JSON object: recording name -> floor height")
    for p in (a, v):
        p.add_argument("--device", default="cuda:0")
    args = ap.parse_args(argv)

    if args.mode == "amass":
        with open(args.saved_data_path, "rb") as f:
            saved = pickle.load(f)
        res = metrics.from_payload(saved, args.mask_scheme, args.traj_mask_ratio, device=args.device)['all']
        print('mpjpe_global (mm): {:0.1f}'.format(res['mpjpe_global'] * 1000))
        print('mpjpe_global_vis / occ (mm): {:0.1f} / {:0.1f}'.format(res['mpjpe_global_vis'] * 1000,
                                                                     res['mpjpe_global_occ'] * 1000))
        print('contact_lbl_acc: {:0.2f}'.format(res['contact_lbl_acc']))
        print('skating_gt_ratio: {:0.3f}'.format(res['skating_gt_ratio']))
        print('skating_rec_ratio: {:0.3f}'.format(res['skating_rec_ratio']))
        print('accel_error (m/s^2): {:0.1f}'.format(res['accel_error']))
        print('ground_pene_freq score (%): {:0.2f}'.format(res['ground_pene_freq'] * 100))
        print('ground_pene_dist score (mm): {:0.2f}'.format(res['ground_pene_dist'] * 1000))
        return

    if args.floor_json:
        with open(args.floor_json) as f:
            table = json.load(f)
        missing = [r for r in args.recordings if r not in table]
        if missing:
            ap.error(f"--floor_json has no floor height for {missing}")
        floors = [float(table[r]) for r in args.recordings]
    else:
        floors = args.floor_height
        if len(floors) != len(args.recordings):
            ap.error(f"--floor_height needs one height per recording ({len(args.recordings)}), got {len(floors)}")
    payloads = []
    for r in args.recordings:
        with open(os.path.join(args.saved_data_dir, r + ".pkl"), "rb") as f:
            payloads.append(pickle.load(f))
    res = metrics.from_payload(payloads, dataset=args.dataset, floor_height=floors, device=args.device)['all']
    print('\n --------------- evaluation metrics -------------')
    print('skating score: {:0.3f}'.format(res['skating']))
    if args.dataset == 'prox':
        print('||acc|| (m/s^2): {:0.2f}'.format(res['acc']))
    else:
        print('acc errors (m/s^2): {:0.2f}'.format(res['acc_error']))
    print('ground_pene_freq score (%): {:0.2f}'.format(res['ground_pene_freq'] * 100))
    print('ground_pene_dist score (mm): {:0.2f}'.format(-res['ground_pene_dist'] * 1000))
    if args.dataset == 'egobody':
        print('-------------- gmpjpe/mpjpe/mpjpe-vis/mpjpe-occ (mm) --------------')
        print('{:0.2f} / {:0.2f} / {:0.2f} / {:0.2f}'.format(res['gmpjpe'] * 1000, res['mpjpe'] * 1000,
                                                             res['mpjpe_vis'] * 1000, res['mpjpe_occ'] * 1000))


if __name__ == "__main__":
    main()
