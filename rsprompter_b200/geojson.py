"""GeoJSON output of mask polygons, for loading results into a GIS or drawing them over the image.

A result set becomes a FeatureCollection with one Feature per result dict: its ``properties`` are the dict's fields
(without the RLE ``segmentation``), its ``geometry`` a MultiPolygon of the mask's outlines.  Each polygon is one outer
border (cv2.RETR_CCOMP's top level) followed by the borders of its holes, as traced with CHAIN_APPROX_SIMPLE.
Coordinates are pixel indices: x = column, y = row of a border pixel, no georeferencing and no half-pixel shift.
Every ring is closed by repeating its first point.

A border of fewer than 3 distinct points (a single pixel, a one-pixel line) cannot form a valid ring: it is left out,
and an outer border left out takes its holes with it.  A mask with no valid ring gets ``"geometry": null``."""
from __future__ import annotations


def _ring(points) -> list | None:
    """int32 [k, 2] -> a closed ring [[x, y], ...], or None below 3 distinct points."""
    pts = points.tolist()
    if len({(x, y) for x, y in pts}) < 3:
        return None
    return pts + [pts[0]]


def multipolygon(contours: list, hierarchy) -> dict | None:
    """One mask's (contours, hierarchy) (cv2.RETR_CCOMP) -> a GeoJSON MultiPolygon geometry, or None."""
    if hierarchy is None:
        return None
    polys, cur = [], None
    for c, (_, _, _, parent) in zip(contours, hierarchy.reshape(-1, 4).tolist()):
        ring = _ring(c)
        if parent < 0:                      # an outer border: its holes follow it in the list
            cur = [ring] if ring is not None else None
            if cur is not None:
                polys.append(cur)
        elif cur is not None and ring is not None:
            cur.append(ring)
    return dict(type="MultiPolygon", coordinates=polys) if polys else None


def feature_collection(properties: list, polygons: list) -> dict:
    """properties: one dict per result; polygons: its mask's (contours, hierarchy), same order -> FeatureCollection."""
    if len(properties) != len(polygons):
        raise ValueError(f"{len(properties)} results but {len(polygons)} polygon sets")
    return dict(type="FeatureCollection",
                features=[dict(type="Feature", properties=p, geometry=multipolygon(c, h))
                          for p, (c, h) in zip(properties, polygons)])
