"""Collect measured parity errors into the JSON file named by B2D_PARITY_REPORT (to calibrate tolerances); nothing is
written when it is unset."""
import json
import os

PATH = os.environ.get("B2D_PARITY_REPORT")


def record(test, **metrics):
    if not PATH:
        return
    try:
        os.makedirs(os.path.dirname(os.path.abspath(PATH)), exist_ok=True)
        data = {}
        if os.path.isfile(PATH):
            try:
                with open(PATH) as f:
                    data = json.load(f)
            except Exception:
                data = {}
        def plain(v):
            try:
                return float(v)
            except Exception:
                return str(v)
        data[test] = {k: plain(v) for k, v in metrics.items()}
        tmp = PATH + ".tmp"
        with open(tmp, "w") as f:
            json.dump(data, f, indent=1, sort_keys=True)
        os.replace(tmp, PATH)
    except Exception:
        pass
