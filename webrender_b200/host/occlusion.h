// occlusion.h — occlusion culling of axis-aligned rects given front to back, the way the reference's
// compositor culls picture-cache tiles (webrender/src/rectangle_occlusion.rs, FrontToBackBuilder).
//
// Each added rect is cut by every opaque rect added before it; what is left of it is appended, as up
// to four pieces per occluder, to the opaque or the alpha list.  Opaque pieces never overlap one
// another, so the opaque list can be drawn in any order; the alpha list is drawn back to front after
// it.  Pieces are horizontal bands above and below the occluder and the spans left and right of it,
// which keeps rows long.
#pragma once
#include <stddef.h>

#include <vector>

namespace wr {

struct DeviceBox2D {  // units.rs DeviceBox2D: min/max corners in device pixels
  float x0 = 0, y0 = 0, x1 = 0, y1 = 0;
  bool is_empty() const { return !(x1 > x0 && y1 > y0); }
  bool intersects(const DeviceBox2D& o) const { return x0 < o.x1 && o.x0 < x1 && y0 < o.y1 && o.y0 < y1; }
  DeviceBox2D intersection_unchecked(const DeviceBox2D& o) const {
    DeviceBox2D r;
    r.x0 = x0 > o.x0 ? x0 : o.x0; r.y0 = y0 > o.y0 ? y0 : o.y0;
    r.x1 = x1 < o.x1 ? x1 : o.x1; r.y1 = y1 < o.y1 ? y1 : o.y1;
    return r;
  }
  // the smallest box holding both; an empty box adds nothing (euclid Box2D::union)
  DeviceBox2D union_with(const DeviceBox2D& o) const {
    if (o.is_empty()) return *this;
    if (is_empty()) return o;
    DeviceBox2D r;
    r.x0 = x0 < o.x0 ? x0 : o.x0; r.y0 = y0 < o.y0 ? y0 : o.y0;
    r.x1 = x1 > o.x1 ? x1 : o.x1; r.y1 = y1 > o.y1 ? y1 : o.y1;
    return r;
  }
};

namespace occlusion {

struct Item {
  DeviceBox2D rectangle;
  size_t key;
};

// Replace every rect of `rects` that `occ` overlaps by the parts of it outside `occ`.
inline void apply_occluder(const DeviceBox2D& occ, std::vector<DeviceBox2D>& rects) {
  // Walk backwards: pieces appended at the back are not visited again, and the rect they replace is
  // filled with the last entry.
  for (size_t i = rects.size(); i-- > 0;) {
    const DeviceBox2D r = rects[i];
    if (!r.intersects(occ)) continue;
    const float band_y0 = r.y0 > occ.y0 ? r.y0 : occ.y0, band_y1 = r.y1 < occ.y1 ? r.y1 : occ.y1;
    if (r.y0 < occ.y0) rects.push_back(DeviceBox2D{r.x0, r.y0, r.x1, occ.y0});  // above
    if (r.y1 > occ.y1) rects.push_back(DeviceBox2D{r.x0, occ.y1, r.x1, r.y1});  // below
    if (r.x0 < occ.x0) rects.push_back(DeviceBox2D{r.x0, band_y0, occ.x0, band_y1});  // left, occluder's rows
    if (r.x1 > occ.x1) rects.push_back(DeviceBox2D{occ.x1, band_y0, r.x1, band_y1});  // right, occluder's rows
    rects[i] = rects.back();
    rects.pop_back();
  }
}

class FrontToBackBuilder {
 public:
  // Add a rect behind everything added so far.  Returns whether any part of it is visible.
  bool add(const DeviceBox2D& rect, bool is_opaque, size_t key) {
    std::vector<DeviceBox2D> pieces = visible_parts(rect);
    std::vector<Item>& list = is_opaque ? opaque_items_ : alpha_items_;
    for (const DeviceBox2D& p : pieces) list.push_back(Item{p, key});
    return !pieces.empty();
  }
  // Whether any part of `rect` would be visible, without adding it.
  bool test(const DeviceBox2D& rect) const { return !visible_parts(rect).empty(); }
  const std::vector<Item>& opaque_items() const { return opaque_items_; }  // front to back
  const std::vector<Item>& alpha_items() const { return alpha_items_; }    // front to back

 private:
  std::vector<DeviceBox2D> visible_parts(const DeviceBox2D& rect) const {
    std::vector<DeviceBox2D> pieces{rect};
    for (const Item& it : opaque_items_) {
      if (pieces.empty()) break;
      if (it.rectangle.intersects(rect)) apply_occluder(it.rectangle, pieces);
    }
    return pieces;
  }
  std::vector<Item> opaque_items_, alpha_items_;
};

}  // namespace occlusion
}  // namespace wr
