"""Stand-in for plyfile (absent offline) so that the reference's src/model/ply_export.py imports and runs.
`PlyData.write` writes no file: it appends (path, the vertex element's structured array) to `PlyData.written`."""


class PlyElement:
    def __init__(self, data, name):
        self.data, self.name = data, name

    @staticmethod
    def describe(data, name):
        return PlyElement(data, name)


class PlyData:
    written = []

    def __init__(self, elements):
        self.elements = list(elements)

    def write(self, path):
        (vertex,) = self.elements
        PlyData.written.append((path, vertex.data))
