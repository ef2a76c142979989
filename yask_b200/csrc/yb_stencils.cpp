// Registry of built-in solutions: the engine-side counterpart of the reference's REGISTER_SOLUTION
// table (/root/reference/src/compiler/compiler_main.cpp:157-234 looks solutions up by "-stencil").
#include "yb_core.h"

namespace yb {

// emitter-generated solutions (yb_gen.cu)
int gen_registry_size();
const char* gen_registry_name(int i);
int gen_registry_create(const std::string& name, int elem_bytes, StencilSpec& spec, std::unique_ptr<Engine>& eng);

namespace {
struct Entry { const char* name; int default_radius; };
const Entry kEntries[] = {
    {"iso3dfd", 8},
};
}  // namespace

const int kNumBuiltin = int(sizeof(kEntries) / sizeof(kEntries[0]));
int registry_size() { return kNumBuiltin + gen_registry_size(); }
const char* registry_name(int i) {
    if (i < 0 || i >= registry_size()) return "";
    return i < kNumBuiltin ? kEntries[i].name : gen_registry_name(i - kNumBuiltin);
}

int registry_create(const std::string& name, int radius, int elem_bytes, StencilSpec& spec, std::unique_ptr<Engine>& eng) {
    if (name == "iso3dfd") {
        if (radius <= 0) radius = 8;
        if (elem_bytes == 0) elem_bytes = 4;
        if (radius > 8) return set_error(YB_EUNSUPPORTED, "iso3dfd: radius %d > 8 is not supported", radius);
        if (elem_bytes == 8 && (radius == 8 || radius == 3)) {
            // double precision at radius 8 and radius 3 (the radius of the reference's own fp64 validation run,
            // /root/reference/src/kernel/Makefile:1155): emitter-generated sweep kernels.  The other radii take the
            // hand-written engine's fp64 sweep below.
            int rc = gen_registry_create(radius == 8 ? "iso3dfd_fp64" : "iso3dfd_fp64_r3", 8, spec, eng);
            if (rc == 0) { spec.name = "iso3dfd"; spec.radius = radius; }
            return rc;
        }
        spec = iso3dfd_spec(radius, elem_bytes, false);
        eng = make_iso3dfd_engine();
        return 0;
    }
    if (name == "iso3dfd_sponge") {
        // Its default radius in each precision stays on the emitter-generated kernels: 8 in fp32, and in fp64 6, the reference's
        // fp64 validation run of this solution (src/kernel/Makefile:1156).  Every other radius up to 8 takes the hand-written
        // iso3dfd sweep in its sponge form.
        const bool f64 = elem_bytes == 8;
        if (radius > 8) return set_error(YB_EUNSUPPORTED, "iso3dfd_sponge: radius %d > 8 is not supported", radius);
        if (radius <= 0 || radius == (f64 ? 6 : 8)) {
            if (!f64) return gen_registry_create(name, elem_bytes, spec, eng);
            int rc = gen_registry_create("iso3dfd_sponge_fp64_r6", 8, spec, eng);
            if (rc == 0) { spec.name = "iso3dfd_sponge"; spec.radius = 6; }
            return rc;
        }
        if (elem_bytes == 0) elem_bytes = 4;
        if (elem_bytes != 4 && elem_bytes != 8) return set_error(YB_EUNSUPPORTED, "iso3dfd_sponge: elements must be 4 or 8 bytes");
        spec = iso3dfd_spec(radius, elem_bytes, true);
        eng = make_iso3dfd_engine();
        return 0;
    }
    if (const int shape = avepts_shape(name); shape >= 0) {
        // 3axis, 3axis_with_diags, 3plane and cube: the emitter generated them in fp32 at the reference's default radii (4, 4, 3
        // and 2: the constructors' defaults in its src/stencils/SimpleStencils.cpp), which stay on those kernels.  Every other radius up
        // to 8, and every radius in fp64, takes the hand-written average-of-points sweep (yb_avepts.cu).
        static const int default_radius[4] = {4, 4, 3, 2};
        if (radius > 8) return set_error(YB_EUNSUPPORTED, "%s: radius %d > 8 is not supported", name.c_str(), radius);
        const int eb = elem_bytes == 0 ? 4 : elem_bytes;
        if (eb != 4 && eb != 8) return set_error(YB_EUNSUPPORTED, "%s: elements must be 4 or 8 bytes", name.c_str());
        if (eb == 4 && (radius <= 0 || radius == default_radius[shape])) return gen_registry_create(name, elem_bytes, spec, eng);
        spec = avepts_spec(shape, radius <= 0 ? default_radius[shape] : radius, eb);
        eng = make_avepts_engine();
        return 0;
    }
    int rc = gen_registry_create(name, elem_bytes, spec, eng);
    if (rc != YB_EINVAL) return rc;
    return set_error(YB_EINVAL, "unknown stencil solution '%s'", name.c_str());
}

}  // namespace yb
