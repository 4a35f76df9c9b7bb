class Unavailable:
    """Stands in for a cityscapesscripts class: importable, raises when used."""

    def __init__(self, *args, **kwargs):
        raise NotImplementedError(f"{type(self).__name__}: cityscapesscripts is not installed (only the reference's "
                                  "'3ddet' task needs it)")
