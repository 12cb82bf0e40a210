// guik/viewer/light_viewer.hpp STAND-IN for the bag pin (test infrastructure): the viewer calls compile and do nothing.
#pragma once
#include <memory>
#include <string>
namespace guik {
struct ShaderSetting {
  ShaderSetting& set_point_scale(float) { return *this; }
};
inline ShaderSetting Rainbow() { return {}; }
inline ShaderSetting FlatOrange() { return {}; }
inline std::string anon() { return "anon"; }
class LightViewer {
public:
  static LightViewer* instance() {
    static LightViewer v;
    return &v;
  }
  void clear_drawables() {}
  template <class... A>
  void update_drawable(const A&...) {}
  void spin_once() {}
};
}  // namespace guik
