// env.hpp — the CRO_* tuning knobs, validated.
//
// The reference validates every environment value it reads and refuses to
// start on anything else, with one wording
// (internal/controller/composableresource_adapter.go:42-45, :64, :67):
//     the env variable DEVICE_RESOURCE_TYPE has an invalid value: '<v>'
// The probe library follows that convention for its own knobs: each one is
// declared here with its legal range, parsed strictly (decimal digits only, no
// sign, no trailing text) ONCE per cro_probe_init, and an illegal value fails
// the init with the reference's sentence instead of being fed to atoi().
// The values a context was created with are its own (cro_ctx::knobs): a later
// change of the environment, another context or a cro_validate_env call never
// reaches a live context.
#pragma once
#include <string>

namespace cro {
namespace env {

struct Knob {
    const char* name;
    unsigned lo, hi, dflt;
    unsigned multiple_of;   // 0 = any
    const char* what;
};

// Every knob the library reads.  n_out receives the count.
const Knob* table(int* n_out);

// Largest tile * stages of a shared-memory ring (CRO_TMA_READ_*, CRO_TMA_COPY_*, CRO_FUSED_*).  An sm_90 CTA may own
// 232448 bytes of shared memory (227 KiB); the ring kernels' static shared memory (barriers, tile table, the
// reduction's staging: 1280 bytes today) takes some of it.  2 KiB are kept for that, so the ceiling is 225 KiB.
// plan_kernels checks the same sum against the device with the kernels' actual static size.
constexpr unsigned kRingMaxBytes = 225u * 1024u;

// "the env variable <NAME> has an invalid value: '<text>'"
std::string refusal(const char* name, const std::string& text);

// Strict parse of one value against one knob.  Returns false and fills *err with refusal() on anything illegal.
bool parse(const Knob& k, const char* text, unsigned* out, std::string* err);

// One validated reading of every knob.  Default-constructed: every knob at its default.
class Values {
   public:
    Values();
    // Value of a knob.  Every name used in the code base is in table(); an unknown one answers 0.
    unsigned get(const char* name) const;

   private:
    friend bool read(Values* out, std::string* err);
    static constexpr int kMax = 48;
    unsigned v_[kMax];
};

// Reads every knob from the process environment (unset or empty = default) and checks the rings against
// kRingMaxBytes.  False + *err on the first illegal one, and *out is left as it was.  Commits nothing anywhere else.
bool read(Values* out, std::string* err);

}  // namespace env
}  // namespace cro
