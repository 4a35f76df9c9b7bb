from ._stub import Unavailable


class CsBbox3d(Unavailable):
    pass
