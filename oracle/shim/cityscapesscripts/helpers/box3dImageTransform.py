from ._stub import Unavailable

CRS_V, CRS_C, CRS_S = "V", "C", "S"


class Camera(Unavailable):
    pass


class Box3dImageTransform(Unavailable):
    pass
