"""mAP accounting (SURVEY 8f row 4): yb_map_evaluate against the reference's validate_detector_map
(additionally.c:4541-4898) on a small synthetic dataset -- BMP images + label files on disk, the reference's own CPU
forward and decoder on both sides, so only the bookkeeping under test differs."""
import os
import re

import numpy as np
import pytest

import ybtest_util as util

pytestmark = pytest.mark.skipif(not util.have_ref(), reason="reference build absent")


@pytest.mark.parametrize("name,iou_thresh", [("tiny64", 0.5), ("v3_32", 0.5), ("tiny64", 0.75)])
def test_map_accounting_equals_reference(name, iou_thresh, workdir):
    util.check_map_accounting(name, iou_thresh, workdir)


def test_dataset_reader_matches_what_the_reference_reads(workdir):
    """BMP / PPM decode, the label-path rewriting and the label parser of yolo2_light_b200.dataset on the files the
    mAP parity test writes: the reference's loader must see the same pixels (its resize of them == ours of them)."""
    from yolo2_light_b200 import dataset
    from oracle import ref
    root = os.path.join(workdir, "reader")
    os.makedirs(os.path.join(root, "images"), exist_ok=True)
    os.makedirs(os.path.join(root, "labels"), exist_ok=True)
    rng = np.random.default_rng(3)
    for w, h in ((80, 72), (33, 50)):                       # a width whose rows need BMP padding, too
        img = rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
        p = os.path.join(root, "images", f"i{w}.bmp")
        util.write_bmp(p, img)
        assert np.array_equal(dataset.read_image_u8(p), img)
        ppm = os.path.join(root, "images", f"i{w}.ppm")
        open(ppm, "wb").write(b"P6\n# c\n%d %d\n255\n" % (w, h) + img.tobytes())
        assert np.array_equal(dataset.read_image_u8(ppm), img)
        assert dataset.label_path(p) == os.path.join(root, "labels", f"i{w}.txt")
    lab = os.path.join(root, "labels", "i80.txt")
    open(lab, "w").write("3 0.5 0.25 0.125 0.0625\n7 0.1 0.2 0.3 0.4\n")
    got = dataset.read_labels(lab)
    assert got.shape == (2, 5) and got[1, 0] == 7 and np.allclose(got[0], [3, 0.5, 0.25, 0.125, 0.0625])
    assert dataset.read_labels(os.path.join(root, "labels", "missing.txt")).shape == (0, 5)
    open(os.path.join(root, "valid.txt"), "w").write(os.path.join(root, "images", "i80.bmp") + "\n")
    open(os.path.join(root, "names.txt"), "w").write("a\nb\n")
    open(os.path.join(root, "d.cfg"), "w").write(f"classes= 2\nvalid  = {root}/valid.txt\nnames = {root}/names.txt\n# x\n")
    paths, names, truth = dataset.load_validation_set(os.path.join(root, "d.cfg"))
    assert len(paths) == 1 and names == ["a", "b"] and truth.shape == (2, 6) and truth[1, 1] == 7


def test_map_driver_loop_equals_reference_end_to_end(workdir):
    """dataset.evaluate_map (the loop of tools/map.py) with the forward + decoder supplied by the reference through a
    stand-in object: same files in, same mAP out as validate_detector_map.  (The GPU stand-ins of the two calls are
    parity-tested on their own: test_gpu_detect.py, test_device_input_pipeline_bit_exact.)"""
    import yolo2_light_b200 as yb
    from yolo2_light_b200 import dataset
    from oracle import ref
    name = "tiny64"
    cfg, wts = util.model_files(name, workdir)
    rnet = ref.RefNet(cfg, wts, 1, 0, 7)
    classes = rnet.layers[-1]["classes"]
    root = os.path.join(workdir, "mapset_tiny64_50")          # written by test_map_accounting_equals_reference
    if not os.path.exists(os.path.join(root, "data.cfg")):
        util.check_map_accounting(name, 0.5, workdir)
    paths, names, truth = dataset.load_validation_set(os.path.join(root, "data.cfg"))
    assert len(paths) == 7 and len(names) == classes and truth.shape[0] > 0

    class RefBacked:
        batch = 2                                               # exercises the padded last batch (7 images)

        def predict_image_u8(self, imgs, quantized=False):
            self.imgs = imgs

        def detect(self, w, h, thresh, nms, relative=1, letter=0, max_rows=1024, quantized=False):
            dets = []
            for im in self.imgs:
                rnet.predict(ref.load_resize_u8(im, rnet.width, rnet.height)[None])
                dets.append(np.delete(rnet.get_boxes(w, h, thresh, nms), 5, axis=1))
            return dets, np.array([d.shape[0] for d in dets], np.int32)

    mAP, aps, st = dataset.evaluate_map(RefBacked(), paths, truth, classes, 0.5, 0.24)
    out = open(os.path.join(root, "ref_stdout.txt")).read()
    map_ref = float(re.search(r"mean average precision \(mAP\) = ([0-9.]+)", out).group(1))
    tp, fp, fn = re.search(r"TP = (\d+), FP = (\d+), FN = (\d+)", out).groups()
    assert abs(mAP - map_ref) < 5e-7
    assert (int(st["tp"]), int(st["fp"]), int(st["fn"])) == (int(tp), int(fp), int(fn))


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_map_driver_on_the_gpu_equals_validate_detector_map(precision, workdir):
    """SURVEY 8f row 4 on the device: dataset.evaluate_map with the REAL Network -- u8 frames -> yb_network_predict_image_u8
    (device resize) -> forward -> yb_network_detect (device decode + NMS) -> yb_map_evaluate -- on the on-disk dataset the
    reference's validate_detector_map (src/additionally.c:4541-4898) was run on: same TP / FP / FN, same mAP."""
    import yolo2_light_b200 as yb
    from yolo2_light_b200 import dataset
    name = "tiny64"
    cfg, wts = util.model_files(name, workdir)
    root = os.path.join(workdir, "mapset_tiny64_50")          # written by test_map_accounting_equals_reference
    if not os.path.exists(os.path.join(root, "ref_stdout.txt")):
        util.check_map_accounting(name, 0.5, workdir)
    paths, names, truth = dataset.load_validation_set(os.path.join(root, "data.cfg"))
    net = yb.load_network(cfg, wts, batch=2)                  # 7 images: exercises the padded last batch
    if precision == "fp32":
        net.set_precision(yb.YB_PREC_FP32)
    classes = len(names)
    mAP, aps, st = dataset.evaluate_map(net, paths, truth, classes, 0.5, 0.24)
    out = open(os.path.join(root, "ref_stdout.txt")).read()
    map_ref = float(re.search(r"mean average precision \(mAP\) = ([0-9.]+)", out).group(1))
    tp, fp, fn = (int(v) for v in re.search(r"TP = (\d+), FP = (\d+), FN = (\d+)", out).groups())
    if precision == "fp32":
        assert abs(mAP - map_ref) < 5e-6
        assert (int(st["tp"]), int(st["fp"]), int(st["fn"])) == (tp, fp, fn)
    else:   # bf16 tensor cores: detections within 1e-3 of the reference's; a borderline box may change sides
        assert abs(mAP - map_ref) < 0.02
        assert abs(int(st["tp"]) - tp) <= 2 and abs(int(st["fn"]) - fn) <= 2
