"""Import a camera calibrated with OpenCV or ROS: read its calibration file and write the camera JSON that every tool here reads
(`--camera_calibration_json`).

    python -m openimucameracalibrator_b200.opencv_to_json --input calib.yaml --output cam.json --fps 30 [--width W --height H]

Two formats are read, with a small parser for the YAML subset they use (no YAML library needed):
  * an OpenCV FileStorage file, YAML (`%YAML:1.0`, `!!opencv-matrix` with rows / cols / dt / data) or JSON, with `camera_matrix` and
    `distortion_coefficients` (or `K` and `D`, as matrices or flat lists) and `image_width` / `image_height`;
  * a ROS `camera_info` YAML, with `camera_matrix`, `distortion_model` (`plumb_bob`, `rational_polynomial`, or `equidistant` / `fisheye`)
    and `distortion_coefficients`.
`--width` / `--height` supply (or override) the image size.

Mapping: f = fx, aspect_ratio = fy / fx, skew = K[0][1], principal point = (K[0][2], K[1][2]).  OpenCV orders the coefficients
D = [k1, k2, p1, p2, k3, k4, k5, k6, s1, s2, s3, s4, tx, ty]:
  * 4 or 5 coefficients write PINHOLE_RADIAL_TANGENTIAL [.., k1, k2, k3, t1 = p1, t2 = p2] (k3 = 0 when absent);
  * 8 write PINHOLE_RATIONAL [.., k1, k2, k3, t1, t2, k4, k5, k6];
  * 12 or 14 (thin prism s1..s4, tilt tx, ty) are read as 8 when every extra coefficient is zero, and refused otherwise;
  * OpenCV's fisheye module (4 coefficients k1..k4 on theta, `distortion_model: equidistant` / `fisheye`, or `fisheye_model: 1`) writes
    FISHEYE, whose theta_d = theta (1 + k1 theta^2 + k2 theta^4 + k3 theta^6 + k4 theta^8) is the same model.
cv2.projectPoints ignores K[0][1]; calibrateCamera never estimates it, so it is 0 in the files these tools write.
"""
from __future__ import annotations

import json
import re
from argparse import ArgumentParser

from . import camera_models as cm
from . import io_formats as iof

_THIN_PRISM_TILT = ["s1", "s2", "s3", "s4", "tx", "ty"]


def _scalar(text: str):
    text = text.strip()
    if len(text) >= 2 and text[0] == text[-1] and text[0] in "'\"":
        return text[1:-1]
    try:
        return float(text) if re.search(r"[.eE]|nan|inf", text, re.I) else int(text)
    except ValueError:
        return text


def _flow_list(text: str) -> list:
    body = text.strip()[1:-1].strip()
    return [_scalar(t) for t in body.split(",") if t.strip()] if body else []


def parse_yaml_subset(text: str) -> dict:
    """The block mappings, flow lists (possibly over several lines) and scalars of OpenCV FileStorage and ROS camera_info files.  Tags
    (`!!opencv-matrix`), directives (`%YAML:1.0`), document markers and comments are skipped."""
    root: dict = {}
    stack = [(-1, root)]
    pending = None          # (target dict, key, text so far) of a flow list still open
    for raw in text.splitlines():
        line = raw.split("#", 1)[0].rstrip() if "[" not in raw else raw.rstrip()
        if pending is not None:
            d, key, acc = pending
            acc += " " + line.strip()
            if "]" in acc:
                d[key] = _flow_list(acc[:acc.index("]") + 1]); pending = None
            else:
                pending = (d, key, acc)
            continue
        if not line.strip() or line.lstrip().startswith(("%", "---", "...")):
            continue
        m = re.match(r"^(\s*)([^:\s][^:]*?)\s*:(?:\s+(.*))?$", line)
        if not m:
            raise ValueError(f"cannot read the line {raw.strip()!r}")
        indent, key, value = len(m.group(1)), m.group(2).strip().strip("'\""), (m.group(3) or "").strip()
        while stack[-1][0] >= indent:
            stack.pop()
        d = stack[-1][1]
        if value.startswith("!!"):
            value = value.split(None, 1)[1] if " " in value else ""
        if value == "":
            d[key] = {}
            stack.append((indent, d[key]))
        elif value.startswith("["):
            if "]" in value:
                d[key] = _flow_list(value[:value.index("]") + 1])
            else:
                pending = (d, key, value)
        else:
            d[key] = _scalar(value)
    if pending is not None:
        raise ValueError(f"unterminated list under {pending[1]!r}")
    return root


def read_calibration(path: str) -> dict:
    """An OpenCV FileStorage (YAML or JSON) or ROS camera_info file -> its mapping."""
    with open(path) as f:
        text = f.read()
    if text.lstrip().startswith("{"):
        return json.loads(text)
    return parse_yaml_subset(text)


def _values(doc: dict, *keys):
    for k in keys:
        if k in doc:
            v = doc[k]
            if isinstance(v, dict):
                if "data" not in v:
                    raise ValueError(f"`{k}` has no data")
                v = v["data"]
            if not isinstance(v, list) or not all(isinstance(x, (int, float)) for x in v):
                raise ValueError(f"`{k}` must hold a list of numbers")
            return [float(x) for x in v]
    return None


def camera_intrinsics(doc: dict):
    """(model id, Theia-ordered intrinsics) of an OpenCV / ROS calibration mapping."""
    K = _values(doc, "camera_matrix", "K", "k")
    if K is None or len(K) != 9:
        raise ValueError("expected a 3x3 `camera_matrix` (or `K`)")
    if K[3] != 0.0 or K[6] != 0.0 or K[7] != 0.0 or K[8] != 1.0 or not K[0] > 0.0 or not K[4] > 0.0:
        raise ValueError(f"camera matrix {K} is not [[fx, s, cx], [0, fy, cy], [0, 0, 1]] with fx, fy > 0")
    D = _values(doc, "distortion_coefficients", "D", "d")
    if D is None:
        raise ValueError("expected `distortion_coefficients` (or `D`)")
    model_name = str(doc.get("distortion_model", "")).lower()
    fisheye = model_name in ("equidistant", "fisheye") or doc.get("fisheye_model") in (1, "1", "true", "True")
    head = [K[0], K[4] / K[0], K[1], K[2], K[5]]
    if fisheye:
        if len(D) != 4:
            raise ValueError(f"a fisheye calibration has 4 coefficients k1..k4, found {len(D)}")
        return cm.FISHEYE, head + D
    if model_name not in ("", "plumb_bob", "rational_polynomial"):
        raise ValueError(f"distortion_model {model_name!r} is not plumb_bob, rational_polynomial or equidistant")
    if len(D) in (4, 5):
        k3 = D[4] if len(D) == 5 else 0.0
        return cm.PINHOLE_RADIAL_TANGENTIAL, head + [D[0], D[1], k3, D[2], D[3]]
    if len(D) in (12, 14):
        extra = {n: v for n, v in zip(_THIN_PRISM_TILT, D[8:]) if v != 0.0}
        if extra:
            raise ValueError("thin-prism / tilt coefficients are not supported: " + ", ".join(f"{n} = {v}" for n, v in extra.items()) + " are not zero")
        D = D[:8]
    if len(D) == 8:
        return cm.PINHOLE_RATIONAL, head + [D[0], D[1], D[4], D[2], D[3], D[5], D[6], D[7]]
    raise ValueError(f"{len(D)} distortion coefficients: expected 4, 5, 8, 12 or 14 (or 4 for a fisheye calibration)")


def camera_document(doc: dict, fps: float, width=None, height=None) -> dict:
    model, k = camera_intrinsics(doc)
    W = width if width is not None else doc.get("image_width", doc.get("width"))
    H = height if height is not None else doc.get("image_height", doc.get("height"))
    if W is None or H is None:
        raise ValueError("the file gives no image size: pass --width and --height")
    return {"fps": float(fps), "image_width": int(W), "image_height": int(H), "intrinsic_type": cm.MODEL_NAMES[model],
            "intrinsics": iof.intrinsics_dict(model, k)}


def main(argv=None) -> dict:
    parser = ArgumentParser("Convert an OpenCV / ROS camera calibration into a camera JSON")
    parser.add_argument("--input", required=True, help="OpenCV FileStorage YAML / JSON or ROS camera_info YAML")
    parser.add_argument("--output", required=True, help="camera JSON to write")
    parser.add_argument("--fps", required=True, type=float, help="camera frame rate (not part of the calibration file)")
    parser.add_argument("--width", type=int, default=None, help="image width [px] (when the file gives none, or to override it)")
    parser.add_argument("--height", type=int, default=None, help="image height [px]")
    args = parser.parse_args(argv)
    try:
        doc = camera_document(read_calibration(args.input), args.fps, args.width, args.height)
    except (OSError, ValueError) as e:
        raise SystemExit(f"opencv_to_json: {e}")
    with open(args.output, "w") as f:
        json.dump(doc, f, indent=4)
    print(f"{doc['intrinsic_type']} camera written to {args.output}: " + " ".join(f"{a}={b}" for a, b in doc["intrinsics"].items()))
    return doc


if __name__ == "__main__":
    main()
