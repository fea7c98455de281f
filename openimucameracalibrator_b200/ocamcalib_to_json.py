"""Import a camera that OCamCalib (Scaramuzza's Omnidirectional Camera Calibration Toolbox) calibrated: read its `calib_results.txt` and
write the camera JSON that every tool here reads (`--camera_calibration_json`), as the SCARAMUZZA model.

    python -m openimucameracalibrator_b200.ocamcalib_to_json --input calib_results.txt --output cam.json --fps 30

`calib_results.txt` holds, each after its comment lines, the direct polynomial `pol` (length first), the inverse polynomial `invpol`
(length first), the centre as "row column" starting from 0, the affine parameters "c d e" and the image size as "height width".
OCamCalib's sensor axes are (row, column) and its optical axis points away from the scene; this project's camera frame is x right (column),
y down (row), z forward.  So a_i = -pol[i], cx = the centre column, cy = the centre row, and c, d, e carry over unchanged.  `invpol` is
not used: the projection here is the exact root of the polynomial.  OCamCalib fixes pol[1] = 0, and the model here stops at degree 4, so
a file with pol[1] != 0 or a higher degree is refused.
"""
from __future__ import annotations

import json
from argparse import ArgumentParser

from . import camera_models as cm
from . import io_formats as iof


def _numbers(line: str) -> list:
    return [float(t) for t in line.split()]


def read_ocamcalib(path: str) -> dict:
    """calib_results.txt -> {"pol", "invpol", "center_row", "center_col", "c", "d", "e", "height", "width"}."""
    with open(path) as f:
        rows = [ln.strip() for ln in f if ln.strip() and not ln.lstrip().startswith("#")]
    if len(rows) < 5:
        raise ValueError(f"{path}: expected the pol, invpol, centre, affine and image-size lines of calib_results.txt, found {len(rows)} data lines")
    pol_line, inv_line, centre, affine, size = (_numbers(r) for r in rows[:5])

    def counted(v, what):
        n = int(v[0]) if v else -1
        if n < 1 or len(v) != n + 1:
            raise ValueError(f"{path}: the {what} line must give its length and then that many coefficients")
        return v[1:]

    pol, invpol = counted(pol_line, "pol"), counted(inv_line, "invpol")
    if len(centre) != 2 or len(affine) != 3 or len(size) != 2:
        raise ValueError(f"{path}: expected 'row column', 'c d e' and 'height width' lines")
    return dict(pol=pol, invpol=invpol, center_row=centre[0], center_col=centre[1], c=affine[0], d=affine[1], e=affine[2],
                height=int(size[0]), width=int(size[1]))


def scaramuzza_intrinsics(ocam: dict) -> list:
    """OCamCalib's model -> SCARAMUZZA's [a0, c, e, cx, cy, a2, a3, a4, d]."""
    pol = list(ocam["pol"])
    if len(pol) < 2 or pol[1] != 0.0:
        raise ValueError("OCamCalib polynomial with pol[1] != 0: the SCARAMUZZA model has no linear term (OCamCalib fixes it to 0)")
    if len(pol) > 5 and any(v != 0.0 for v in pol[5:]):
        raise ValueError(f"OCamCalib polynomial of degree {len(pol) - 1}: the SCARAMUZZA model stops at degree 4")
    if not pol[0] < 0.0:
        raise ValueError("OCamCalib polynomial with pol[0] >= 0: its rays would not leave the camera forwards")
    pol = (pol + [0.0] * 5)[:5]
    return [-pol[0], ocam["c"], ocam["e"], ocam["center_col"], ocam["center_row"], -pol[2], -pol[3], -pol[4], ocam["d"]]


def camera_document(ocam: dict, fps: float) -> dict:
    k = scaramuzza_intrinsics(ocam)
    return {"fps": float(fps), "image_width": int(ocam["width"]), "image_height": int(ocam["height"]), "intrinsic_type": cm.MODEL_NAMES[cm.SCARAMUZZA],
            "intrinsics": iof.intrinsics_dict(cm.SCARAMUZZA, k)}


def main(argv=None) -> dict:
    parser = ArgumentParser("Convert OCamCalib's calib_results.txt into a SCARAMUZZA camera JSON")
    parser.add_argument("--input", required=True, help="OCamCalib calib_results.txt")
    parser.add_argument("--output", required=True, help="camera JSON to write")
    parser.add_argument("--fps", required=True, type=float, help="camera frame rate (not part of OCamCalib's file)")
    args = parser.parse_args(argv)
    try:
        doc = camera_document(read_ocamcalib(args.input), args.fps)
    except (OSError, ValueError) as e:
        raise SystemExit(f"ocamcalib_to_json: {e}")
    with open(args.output, "w") as f:
        json.dump(doc, f, indent=4)
    print(f"SCARAMUZZA camera written to {args.output}: " + " ".join(f"{a}={b}" for a, b in doc["intrinsics"].items()))
    return doc


if __name__ == "__main__":
    main()
