"""Import shim for the reference's `cityscapesscripts` (not installed here). TP/data/cityscapes3d.py:17-24 imports a few
names at module level; only its '3ddet' task (load_det) uses them, and that task is out of scope, so the stubs raise
when called."""
