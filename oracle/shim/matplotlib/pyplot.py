"""Import-only shim (see the package docstring)."""


def imsave(*args, **kwargs):
    raise NotImplementedError("matplotlib is not installed; the reference only calls imsave in dead branches")
