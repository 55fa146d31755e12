"""TEST TOOLING — tests/golden/decode_edges.npz: the UNMODIFIED reference nms_hm / select_topk / PostProcessor
(model/layers/utils.py, model/head/detector_infer.py, via oracle/ref_shims.py) on the cases of oracle/decode_edge_cases.py
listed in GOLDEN_CASES: a clamped background at 96x320 (B = 2), saturated ties, fewer maxima than K. Build container only:

    python -m oracle.make_golden_decode_edges

The maps are not stored; the builder regenerates them and `<case>/checksum` pins its inputs. Per case: the reference's
top-k tensors `<case>/scores`, `inds`, `clses` [B, K] and per image `<case>/result_b<b>` [N, 14] at the case's
threshold. torch.topk leaves the order of ties unspecified, so every case keeps at most K local maxima at or above its
threshold in each image: the set of detections is then fully determined, and only their order among equal scores is not.
The archive is written with fixed member timestamps, so regenerating it gives identical bytes."""
import io
import os
import sys
import zipfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shims as rs                # noqa: E402
from oracle import decode_edge_cases as de        # noqa: E402
from oracle.make_golden import ref_targets        # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "decode_edges.npz")


def save_npz(path, arrays):
    """np.savez_compressed with a fixed member order and timestamp"""
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(arrays[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())


def run_case(name):
    rs.install()
    import model.layers.utils as lu
    case = de.build(name)
    assert not case["apply_sigmoid"]
    heat, reg, K, thr = case["maps"], case["reg"], case["K"], case["thresh"]
    B, C, H, W = heat.shape
    assert int(de.n_above(case).max()) <= K, "%s: more than K detections at or above the threshold" % name
    cfg = rs.reference_cfg(width=4 * W, height=4 * H)
    cfg.TEST.DETECTIONS_PER_IMG = K
    pp = rs.build_reference_model(cfg).eval().heads.post_processor
    pp.det_threshold = thr
    tg = dict(calib_P=case["calib_P"], pad_size=case["pad"], size=[tuple(int(v) for v in s) for s in case["size"]],
              edge_indices=torch.zeros(B, 1, 2, dtype=torch.long), edge_len=torch.zeros(B, dtype=torch.long))
    targets = ref_targets(tg)
    out = {"checksum": np.array(de.checksum(case))}
    with torch.no_grad():
        sc, inds, cls_, _, _ = lu.select_topk(lu.nms_hm(heat.clone()), K)
        out.update(scores=sc.numpy(), inds=inds.numpy(), clses=cls_.numpy())
        for b in range(B):
            res, _, _ = pp({"cls": heat[b:b + 1].clone(), "reg": reg[b:b + 1].clone()}, targets[b:b + 1], test=True)
            out["result_b%d" % b] = res.numpy()
    return out


def main():
    torch.set_num_threads(8)
    out = {}
    for name in de.GOLDEN_CASES:
        res = run_case(name)
        out.update({"%s/%s" % (name, k): v for k, v in res.items()})
        print("%-10s detections per image %s" % (name, [out["%s/result_b%d" % (name, b)].shape[0]
                                                        for b in range(res["scores"].shape[0])]))
    save_npz(OUT, out)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
