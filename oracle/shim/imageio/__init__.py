"""Import shim for the reference's `imageio` (not installed here): imwrite writes the array through PIL, which is what
the reference's PNG exports need (evaluate_utils.py save_model_pred_for_one_task)."""


def imwrite(uri, im, *args, **kwargs):
    import numpy as np
    from PIL import Image

    Image.fromarray(np.asarray(im)).save(uri)
