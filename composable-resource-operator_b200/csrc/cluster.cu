// cluster.cu — see cluster.hpp.  (.cu only because it reaches the probe
// context, whose header pulls in CUDA types; there is no device code here.)
#include "cluster.hpp"

#include <algorithm>
#include <unistd.h>

#include <chrono>
#include <cstdio>
#include <cstring>

#include "identity.hpp"
#include "probe.hpp"

namespace cro {
namespace sim {

namespace {
const char* kFinalizer = "com.ie.ibm.hpsys/finalizer";                 // composabilityrequest_controller.go:45
const char* kLastUsed = "cohdi.io/last-used-time";                     // :46
const char* kDeleteDevice = "cohdi.io/delete-device";                  // :47
const char* kManagedBy = "app.kubernetes.io/managed-by";
const char* kReadyToDetach = "cohdi.io/ready-to-detach-device-id";

bool contains(const std::vector<std::string>& v, const std::string& s) {
    return std::find(v.begin(), v.end(), s) != v.end();
}
void removeStr(std::vector<std::string>* v, const std::string& s) {
    v->erase(std::remove(v->begin(), v->end(), s), v->end());
}

// time.Parse(time.RFC3339, s) reduced to a sortable integer (seconds since epoch).
bool parseRFC3339(const std::string& s, long long* out) {
    int Y, M, D, h, m, sec;
    int n = 0;
    if (sscanf(s.c_str(), "%4d-%2d-%2dT%2d:%2d:%2d%n", &Y, &M, &D, &h, &m, &sec, &n) != 6) return false;
    std::string rest = s.substr((size_t)n);
    if (!rest.empty() && rest[0] == '.') {   // fractional seconds
        size_t k = 1;
        while (k < rest.size() && isdigit((unsigned char)rest[k])) ++k;
        if (k == 1) return false;
        rest = rest.substr(k);
    }
    long long off = 0;
    if (rest == "Z") off = 0;
    else if (rest.size() == 6 && (rest[0] == '+' || rest[0] == '-') && rest[3] == ':') {
        off = ((rest[1] - '0') * 10 + (rest[2] - '0')) * 3600 + ((rest[4] - '0') * 10 + (rest[5] - '0')) * 60;
        if (rest[0] == '-') off = -off;
    } else return false;
    // days from civil (Howard Hinnant)
    long long y = Y - (M <= 2);
    const long long era = (y >= 0 ? y : y - 399) / 400;
    const long long yoe = y - era * 400;
    const long long doy = (153 * (M + (M > 2 ? -3 : 9)) + 2) / 5 + D - 1;
    const long long doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
    const long long days = era * 146097 + doe - 719468;
    *out = days * 86400 + h * 3600 + m * 60 + sec - off;
    return true;
}

ScalarResourceDetails detailsFromJson(const gojson::Value* v) {
    ScalarResourceDetails d;
    if (!v) return d;
    d.Type = v->get_string("type");
    d.Model = v->get_string("model");
    d.Size = v->get_int("size");
    d.ForceDetach = v->get_bool("force_detach");
    d.AllocationPolicy = v->get_string("allocation_policy", "samenode");   // CRD default
    d.TargetNode = v->get_string("target_node");
    if (const gojson::Value* o = v->get("other_spec")) {
        if (o->kind == gojson::Value::Object) {
            d.HasOtherSpec = true;
            d.OtherSpec.MilliCPU = o->get_int("milli_cpu");
            d.OtherSpec.Memory = o->get_int("memory");
            d.OtherSpec.EphemeralStorage = o->get_int("ephemeral_storage");
            d.OtherSpec.AllowedPodNumber = o->get_int("allowed_pod_number");
        }
    }
    return d;
}
}  // namespace

// ---- JSON of the API types (declaration order, omitempty as tagged) -----------
std::string ScalarResourceDetails::MarshalJSON() const {
    gojson::Writer w;
    w.begin_object();
    w.field("type", Type).field("model", Model).field("size", Size);
    w.field_omitempty("force_detach", ForceDetach);
    w.field_omitempty("allocation_policy", AllocationPolicy);
    w.field_omitempty("target_node", TargetNode);
    if (HasOtherSpec) {
        w.key("other_spec").begin_object();
        w.field_omitempty("milli_cpu", OtherSpec.MilliCPU).field_omitempty("memory", OtherSpec.Memory);
        w.field_omitempty("ephemeral_storage", OtherSpec.EphemeralStorage);
        w.field_omitempty("allowed_pod_number", OtherSpec.AllowedPodNumber);
        w.end_object();
    }
    w.end_object();
    return w.take();
}
std::string ScalarResourceStatus::MarshalJSON() const {
    gojson::Writer w;
    w.begin_object();
    w.field("state", State);
    w.field_omitempty("device_id", DeviceID).field_omitempty("cdi_device_id", CDIDeviceID);
    w.field_omitempty("node_name", NodeName).field_omitempty("error", Error);
    w.end_object();
    return w.take();
}
std::string ComposabilityRequestStatus::MarshalJSON() const {
    gojson::Writer w;
    w.begin_object();
    w.field("state", State);
    w.field_omitempty("error", Error);
    if (!Resources.empty()) {   // omitempty on the map
        w.key("resources").begin_object();
        for (const auto& kv : Resources) w.key(kv.first.c_str()).raw(kv.second.MarshalJSON());
        w.end_object();
    }
    w.key("scalarResource").raw(ScalarResource.MarshalJSON());   // struct: omitempty never drops it
    w.end_object();
    return w.take();
}

// ---- construction ----------------------------------------------------------------
Cluster::Cluster(cro_ctx* ctx, const gojson::Value& cfg) : ctx_(ctx), rng_(20260921) {
    deviceResourceType_ = cfg.get_string("device_resource_type", "DEVICE_PLUGIN");
    probe_ = cfg.get_bool("probe") && ctx != nullptr;
    stats.tracing = cfg.get_bool("trace");
    if (cfg.get("seed")) rng_.seed((unsigned long long)cfg.get_int("seed"));
    if (const gojson::Value* ns = cfg.get("nodes"))
        for (const auto& n : ns->arr) {
            Node node;
            if (n->kind == gojson::Value::String) {
                node.Name = n->str;
                node.CPU = 8; node.Memory = 16ll << 30; node.EphemeralStorage = 512ll << 30; node.Pods = 100;
            } else {
                node.Name = n->get_string("name");
                node.CPU = n->get_int("cpu"); node.Memory = n->get_int("memory");
                node.EphemeralStorage = n->get_int("ephemeral_storage"); node.Pods = n->get_int("pods");
            }
            nodes_.push_back(node);
        }
    std::sort(nodes_.begin(), nodes_.end(), [](const Node& a, const Node& b) { return a.Name < b.Name; });
    if (const gojson::Value* us = cfg.get("uuids"))
        for (const auto& u : us->arr)
            if (u->kind == gojson::Value::String) uuids_.push_back(u->str);
    if (uuids_.empty() && ctx)
        for (auto& d : ctx->devs) uuids_.push_back(std::string(d->info.gpu_uuid, strnlen(d->info.gpu_uuid, 48)));
    if (probe_ && ctx) {
        // "warm probe contexts" (SURVEY.md §8d config 4): both lanes of every device run once before the clock starts, so
        // no graph capture / instantiation (milliseconds of host time each) falls into the reconcile loop
        for (size_t i = 0; i < ctx->devs.size(); ++i) { ctx_probe_begin(ctx, (int)i); ctx_probe_begin(ctx, (int)i); }
        for (size_t i = 0; i < ctx->devs.size(); ++i) {
            cro_probe_result warm;
            ctx_probe_end(ctx, (int)i, &warm);
            ctx_probe_end(ctx, (int)i, &warm);
        }
    }
    if (uuids_.empty()) uuids_.push_back("GPU-00000000-0000-0000-0000-000000000000");
}

const Node* Cluster::getNode(const std::string& name) const {
    for (const Node& n : nodes_)
        if (n.Name == name) return &n;
    return nullptr;
}

// internal/utils/nodes.go:78-117.  Quirk kept: MilliCPU is compared with the
// node's WHOLE cores (AsInt64), SURVEY.md Appendix A-8.
Error Cluster::CheckNodeCapacitySufficient(const std::string& nodeName, const NodeSpec& spec, bool* ok) const {
    const Node* n = getNode(nodeName);
    if (!n) return Error::New("nodes \"" + nodeName + "\" not found");
    *ok = !(n->CPU < spec.MilliCPU || n->Memory < spec.Memory || n->Pods < spec.AllowedPodNumber ||
            n->EphemeralStorage < spec.EphemeralStorage);
    return Error::Nil();
}

// internal/utils/stringutils.go:26-33 — "<type>-<uuid4>", lower case
std::string Cluster::GenerateComposableResourceName(const std::string& typeName) {
    unsigned long long a = rng_(), b = rng_();
    a = (a & 0xFFFFFFFFFFFF0FFFull) | 0x0000000000004000ull;   // version 4
    b = (b & 0x3FFFFFFFFFFFFFFFull) | 0x8000000000000000ull;   // variant 10
    char buf[64];
    snprintf(buf, sizeof buf, "%08llx-%04llx-%04llx-%04llx-%012llx", a >> 32, (a >> 16) & 0xFFFF, a & 0xFFFF, b >> 48,
             b & 0xFFFFFFFFFFFFull);
    return identity::ToLower(typeName + "-" + buf);
}

// ---- store -------------------------------------------------------------------------
void Cluster::enqueueRequest(const std::string& key) {
    if (req_queued_.insert(key).second) req_queue_.push_back(key);
}
void Cluster::enqueueResource(const std::string& key) {
    if (res_queued_.insert(key).second) res_queue_.push_back(key);
}
// GPU wake-ups jump the queue: a finished probe (or a freed device) should not idle behind
// thousands of unrelated reconciles.
void Cluster::enqueueResourceFront(const std::string& key) {
    if (res_queued_.insert(key).second) { res_queue_.push_front(key); return; }
    auto it = std::find(res_queue_.begin(), res_queue_.end(), key);
    if (it != res_queue_.end() && it != res_queue_.begin()) { res_queue_.erase(it); res_queue_.push_front(key); }
}

void Cluster::updateRequest(const ComposabilityRequest& r) {
    auto it = requests_.find(r.Name);
    if (it == requests_.end()) return;   // NotFound
    const ComposabilityRequest& old = it->second;
    const bool changed = !(old.Status == r.Status) || !(old.Spec == r.Spec) || old.Finalizers != r.Finalizers ||
                         old.DeletionTimestampSet != r.DeletionTimestampSet;
    // r.Update (finalizers) comes before r.Status().Update in every handler that does both
    if (!fault_update_.empty() && (old.Finalizers != r.Finalizers || !(old.Spec == r.Spec))) throw ApiFault{fault_update_};
    if (!fault_status_update_.empty() && !(old.Status == r.Status)) throw ApiFault{fault_status_update_};
    if (!(old.Status == r.Status)) {   // Status().Update marshals the status: one emitted spec
        ++stats.status_updates;
        stats.spec_bytes += (long long)r.Status.MarshalJSON().size();
    }
    if (!changed) return;
    ++changes_;
    it->second = r;
    if (r.DeletionTimestampSet && r.Finalizers.empty()) {
        requests_.erase(it);
        return;
    }
    enqueueRequest(r.Name);
}

void Cluster::deleteRequest(const std::string& name) {
    auto it = requests_.find(name);
    if (it == requests_.end()) return;
    ++changes_;
    if (it->second.Finalizers.empty()) {
        requests_.erase(it);
        return;
    }
    if (!it->second.DeletionTimestampSet) {
        it->second.DeletionTimestampSet = true;
        enqueueRequest(name);
    }
}

void Cluster::createResource(const StoredResource& r) {
    StoredResource s = r;
    s.CreationSeq = ++seq_;
    resources_[s.obj.Name] = s;
    ++changes_;
    enqueueResource(s.obj.Name);   // the request controller's predicate drops Create events (:669)
}

void Cluster::updateResource(const StoredResource& r) {
    auto it = resources_.find(r.obj.Name);
    if (it == resources_.end()) return;
    const StoredResource& old = it->second;
    const bool status_changed = old.obj.Status.State != r.obj.Status.State || old.obj.Status.Error != r.obj.Status.Error ||
                                old.obj.Status.DeviceID != r.obj.Status.DeviceID ||
                                old.obj.Status.CDIDeviceID != r.obj.Status.CDIDeviceID;
    const bool changed = status_changed || old.Finalizers != r.Finalizers || old.obj.Labels != r.obj.Labels ||
                         old.Annotations != r.Annotations || old.obj.DeletionTimestampSet != r.obj.DeletionTimestampSet;
    if (!fault_update_.empty() && (old.Finalizers != r.Finalizers || old.obj.Labels != r.obj.Labels || old.Annotations != r.Annotations))
        throw ApiFault{fault_update_};
    if (!fault_status_update_.empty() && status_changed) throw ApiFault{fault_status_update_};
    if (status_changed) {
        ++stats.status_updates;
        stats.spec_bytes += (long long)r.obj.Status.MarshalJSON().size();
    }
    if (!changed) return;
    ++changes_;
    const long long seq = old.CreationSeq;
    it->second = r;
    it->second.CreationSeq = seq;
    if (status_changed) enqueueRequest(r.obj.Name);   // resourceStatusUpdatePredicate (:658-667)
    if (r.obj.DeletionTimestampSet && r.Finalizers.empty()) {
        resources_.erase(it);
        return;
    }
    enqueueResource(r.obj.Name);
}

void Cluster::deleteResource(const std::string& name) {
    auto it = resources_.find(name);
    if (it == resources_.end()) return;
    ++changes_;
    if (it->second.Finalizers.empty()) {
        resources_.erase(it);
        return;
    }
    if (!it->second.obj.DeletionTimestampSet) {
        it->second.obj.DeletionTimestampSet = true;
        enqueueResource(name);
    }
}

// ---- kubectl -------------------------------------------------------------------------
Error Cluster::Apply(const gojson::Value& v) {
    const std::string name = v.get_string("name");
    if (name.empty()) return Error::New("request needs a name");
    const gojson::Value* res = v.get("resource");
    ScalarResourceDetails d = detailsFromJson(res);
    // CRD validation (config/crd/bases/...composabilityrequests.yaml:45-90)
    // The API server's words (apimachinery field.ErrorList -> StatusError), pinned one field at a time by
    // composabilityrequest_controller_test.go:324-412; several bad fields aggregate as "[a, b]" (order unpinned).
    {
        std::vector<std::string> errs;
        auto quoted = [](const std::string& s) { std::string o; gojson::append_string(o, s); return o; };
        auto minimum = [&](const char* path, long long v) {
            if (v < 0)
                errs.push_back(std::string(path) + ": Invalid value: " + std::to_string(v) + ": " + path +
                               " in body should be greater than or equal to 0");
        };
        if (d.Type != "gpu" && d.Type != "cxlmemory")
            errs.push_back("spec.resource.type: Unsupported value: " + quoted(d.Type) + ": supported values: \"gpu\", \"cxlmemory\"");
        if (d.Model.empty())
            errs.push_back("spec.resource.model: Invalid value: \"\": spec.resource.model in body should be at least 1 chars long");
        minimum("spec.resource.size", d.Size);
        if (d.AllocationPolicy != "samenode" && d.AllocationPolicy != "differentnode")
            errs.push_back("spec.resource.allocation_policy: Unsupported value: " + quoted(d.AllocationPolicy) +
                           ": supported values: \"samenode\", \"differentnode\"");
        if (d.HasOtherSpec) {
            minimum("spec.resource.other_spec.milli_cpu", d.OtherSpec.MilliCPU);
            minimum("spec.resource.other_spec.memory", d.OtherSpec.Memory);
            minimum("spec.resource.other_spec.ephemeral_storage", d.OtherSpec.EphemeralStorage);
            minimum("spec.resource.other_spec.allowed_pod_number", d.OtherSpec.AllowedPodNumber);
        }
        if (!errs.empty()) {
            std::string all = errs[0];
            if (errs.size() > 1) {
                all = "[" + errs[0];
                for (size_t i = 1; i < errs.size(); ++i) all += ", " + errs[i];
                all += "]";
            }
            return Error::New("ComposabilityRequest.cro.hpsys.ibm.ie.com \"" + name + "\" is invalid: " + all);
        }
    }
    // validating admission webhook, create and update alike (internal/webhook/v1alpha1/composabilityrequest_webhook.go:
    // validateRequest :100-147); the API server wraps the webhook's message in its own sentence
    {
        const std::string denied = "admission webhook \"vcomposabilityrequest.kb.io\" denied the request: ";
        if (d.AllocationPolicy == "differentnode" && !d.TargetNode.empty())
            return Error::New(denied + "TargetNode cannot be specified when AllocationPolicy is set to 'differentnode'");
        // one request per (type, model) cluster-wide for "differentnode"; one per (node, type, model) for "samenode", where
        // a request without target_node counts for the node its first child landed on ("" while it has none)
        for (const auto& kv : requests_) {        // List() order: by name
            const ComposabilityRequest& o = kv.second;
            if (o.Name == name) continue;
            bool clash = false;
            if (d.AllocationPolicy == "differentnode") {
                clash = o.Spec.AllocationPolicy == "differentnode" && o.Spec.Type == d.Type && o.Spec.Model == d.Model;
            } else if (d.AllocationPolicy == "samenode") {
                std::string targetNode = o.Spec.TargetNode;
                if (targetNode.empty() && !o.Status.Resources.empty()) targetNode = o.Status.Resources.begin()->second.NodeName;
                clash = targetNode == d.TargetNode && o.Spec.Type == d.Type && o.Spec.Model == d.Model;
            }
            if (clash)
                return Error::New(denied + "composabilityRequest resource " + o.Name + " with type " + d.Type + " and model " + d.Model +
                                  " already exists");
        }
    }
    auto it = requests_.find(name);
    if (it == requests_.end()) {
        ComposabilityRequest r;
        r.Name = name;
        r.Spec = d;
        r.CreationSeq = ++seq_;
        requests_[name] = r;
        ++changes_;
        enqueueRequest(name);
    } else {
        ComposabilityRequest r = it->second;
        r.Spec = d;
        updateRequest(r);
    }
    return Error::Nil();
}

Error Cluster::Delete(const std::string& name) {
    if (!requests_.count(name)) return Error::New("composabilityrequests \"" + name + "\" not found");
    deleteRequest(name);
    return Error::Nil();
}

Error Cluster::Plant(const gojson::Value& v) {
    const std::string kind = v.get_string("kind");
    const std::string name = v.get_string("name");
    if (kind == "Fault") {   // arm / clear the API-server faults
        fault_update_ = v.get_string("update");
        fault_status_update_ = v.get_string("status_update");
        return Error::Nil();
    }
    if (kind == "ComposabilityRequest") {
        ComposabilityRequest r;
        r.Name = name;
        r.Spec = detailsFromJson(v.get("resource"));
        r.CreationSeq = ++seq_;
        if (const gojson::Value* st = v.get("status")) {
            r.Status.State = st->get_string("state");
            r.Status.Error = st->get_string("error");
            r.Status.ScalarResource = st->get("scalarResource") ? detailsFromJson(st->get("scalarResource")) : r.Spec;
            if (const gojson::Value* rs = st->get("resources"))
                for (const auto& kv : rs->obj) {
                    ScalarResourceStatus s;
                    s.State = kv.second->get_string("state");
                    s.DeviceID = kv.second->get_string("device_id");
                    s.CDIDeviceID = kv.second->get_string("cdi_device_id");
                    s.NodeName = kv.second->get_string("node_name");
                    s.Error = kv.second->get_string("error");
                    r.Status.Resources[kv.first] = s;
                }
        }
        if (v.get_bool("finalizer", true)) r.Finalizers.push_back(kFinalizer);
        r.DeletionTimestampSet = v.get_bool("deleting");
        requests_[name] = r;
        return Error::Nil();
    }
    if (kind == "ComposableResource") {
        StoredResource s;
        s.obj.Name = name;
        s.CreationSeq = ++seq_;
        if (const gojson::Value* sp = v.get("spec")) {
            s.obj.Spec.Type = sp->get_string("type");
            s.obj.Spec.Model = sp->get_string("model");
            s.obj.Spec.TargetNode = sp->get_string("target_node");
            s.obj.Spec.ForceDetach = sp->get_bool("force_detach");
        }
        if (const gojson::Value* st = v.get("status")) {
            s.obj.Status.State = st->get_string("state");
            s.obj.Status.Error = st->get_string("error");
            s.obj.Status.DeviceID = st->get_string("device_id");
            s.obj.Status.CDIDeviceID = st->get_string("cdi_device_id");
        }
        if (const gojson::Value* lb = v.get("labels"))
            for (const auto& kv : lb->obj) s.obj.Labels[kv.first] = kv.second->str;
        if (const gojson::Value* an = v.get("annotations"))
            for (const auto& kv : an->obj) s.Annotations[kv.first] = kv.second->str;
        if (v.get_bool("finalizer", true)) s.Finalizers.push_back(kFinalizer);
        s.obj.DeletionTimestampSet = v.get_bool("deleting");
        if (!s.obj.Status.DeviceID.empty()) attached_.insert(name);
        resources_[name] = s;
        return Error::Nil();
    }
    return Error::New("unknown kind '" + kind + "'");
}

// =====================================================================================
// ComposabilityRequestReconciler  (internal/controller/composabilityrequest_controller.go)
// =====================================================================================
class RequestReconciler {
public:
    explicit RequestReconciler(Cluster* c) : c_(c) {}

    Error requeueOnErr(ComposabilityRequest* r, const Error& err) {   // :627-637
        // a Go panic never reaches requeueOnErr: it unwinds to controller-runtime's wrapper, no status write on the way
        if (err.panicked() || err.recovered()) return Error::Recovered(err);
        if (r) {
            r->Status.Error = err.msg;
            try { c_->updateRequest(*r); } catch (const ApiFault&) {}   // best effort (:631-634): the original error wins
        }
        return err;
    }

    Error Reconcile(const std::string& key, long long* requeue) {   // :72-96
        *requeue = 0;
        auto it = c_->requests_.find(key);
        if (it != c_->requests_.end()) {
            ComposabilityRequest r = it->second;
            return handleComposabilityRequestChange(&r, requeue);
        }
        auto jt = c_->resources_.find(key);
        if (jt != c_->resources_.end()) return handleComposableResourceChange(jt->second);
        return Error::Nil();   // "could not find the resource": logged, not requeued
    }

private:
    Error handleComposabilityRequestChange(ComposabilityRequest* r, long long* requeue) {   // :98-145
        // performGarbageCollection :147-167
        if (!r->Spec.TargetNode.empty() && !c_->getNode(r->Spec.TargetNode)) {
            if (!r->DeletionTimestampSet) {
                c_->deleteRequest(r->Name);
                return Error::Nil();
            }
        }
        Error err;
        const std::string& st = r->Status.State;
        if (st.empty()) err = handleNoneState(r);
        else if (st == "NodeAllocating") err = handleNodeAllocatingState(r);
        else if (st == "Updating") err = handleUpdatingState(r, requeue);
        else if (st == "Running") err = handleRunningState(r, requeue);
        else if (st == "Cleaning") err = handleCleaningState(r, requeue);
        else if (st == "Deleting") err = handleDeletingState(r);
        else return requeueOnErr(r, Error::New("the composabilityRequest state '" + st + "' is invalid"));
        // handlers already routed their own failures through requeueOnErr
        return err;
    }

    Error handleComposableResourceChange(const StoredResource& child) {   // :169-195
        auto lb = child.obj.Labels.find(kReadyToDetach);
        if (lb != child.obj.Labels.end() && !lb->second.empty()) return Error::Nil();
        auto mb = child.obj.Labels.find(kManagedBy);
        const std::string parent = mb == child.obj.Labels.end() ? std::string() : mb->second;
        auto it = c_->requests_.find(parent);
        if (it == c_->requests_.end())
            return Error::New("composabilityrequests.cro.hpsys.ibm.ie.com \"" + parent + "\" not found");
        ComposabilityRequest r = it->second;
        auto slot = r.Status.Resources.find(child.obj.Name);
        if (slot != r.Status.Resources.end()) {
            slot->second.State = child.obj.Status.State;
            slot->second.Error = child.obj.Status.Error;
            slot->second.DeviceID = child.obj.Status.DeviceID;
            slot->second.CDIDeviceID = child.obj.Status.CDIDeviceID;
        }
        c_->updateRequest(r);
        return Error::Nil();
    }

    Error handleNoneState(ComposabilityRequest* r) {   // :197-211
        if (!contains(r->Finalizers, kFinalizer)) r->Finalizers.push_back(kFinalizer);
        r->Status.State = "NodeAllocating";
        r->Status.Error = "";
        r->Status.ScalarResource = r->Spec;
        c_->updateRequest(*r);
        return Error::Nil();
    }

    std::vector<const StoredResource*> children(const std::string& request, bool filter) const {
        std::vector<const StoredResource*> out;
        for (const auto& kv : c_->resources_) {
            auto mb = kv.second.obj.Labels.find(kManagedBy);
            if (mb == kv.second.obj.Labels.end() || mb->second != request) continue;
            if (filter && (kv.second.obj.Status.State == "Detaching" || kv.second.obj.Status.State == "Deleting")) continue;
            out.push_back(&kv.second);
        }
        return out;
    }

    Error handleNodeAllocatingState(ComposabilityRequest* r) {   // :213-485
        if (r->DeletionTimestampSet) {
            r->Status.State = "Cleaning";
            c_->updateRequest(*r);
            return Error::Nil();
        }
        const std::vector<const StoredResource*> kids = children(r->Name, true);
        long long resourcesToAllocate = r->Spec.Size;
        long long resourcesToDelete = 0;
        std::set<std::string> allocatedNodesForDifferentPolicy;
        std::string targetNodeForSamePolicy;

        for (const StoredResource* k : kids) {   // :254-305
            const controller::ComposableResource& res = k->obj;
            if (resourcesToAllocate > 0) {
                if (res.Spec.Type != r->Spec.Type || res.Spec.Model != r->Spec.Model || res.Spec.ForceDetach != r->Spec.ForceDetach) {
                    r->Status.Resources.erase(res.Name);
                    continue;
                }
                if (!r->Spec.TargetNode.empty() && res.Spec.TargetNode != r->Spec.TargetNode) {
                    r->Status.Resources.erase(res.Name);
                    continue;
                }
                if (r->Spec.HasOtherSpec) {
                    bool ok = false;
                    Error e = c_->CheckNodeCapacitySufficient(res.Spec.TargetNode, r->Spec.OtherSpec, &ok);
                    if (!e.ok()) return requeueOnErr(r, e);
                    if (!ok) {
                        r->Status.Resources.erase(res.Name);
                        continue;
                    }
                }
                if (r->Spec.AllocationPolicy == "differentnode") {
                    if (allocatedNodesForDifferentPolicy.count(res.Spec.TargetNode)) {
                        r->Status.Resources.erase(res.Name);
                        continue;
                    }
                    allocatedNodesForDifferentPolicy.insert(res.Spec.TargetNode);
                } else if (r->Spec.AllocationPolicy == "samenode") {
                    if (targetNodeForSamePolicy.empty()) targetNodeForSamePolicy = res.Spec.TargetNode;
                    else if (targetNodeForSamePolicy != res.Spec.TargetNode) {
                        r->Status.Resources.erase(res.Name);
                        continue;
                    }
                }
                --resourcesToAllocate;
            } else {
                ++resourcesToDelete;
            }
        }

        if (resourcesToDelete > 0) {   // :310-359, the only sort in the reference
            struct P { std::string name; long long key; };
            std::vector<std::vector<P>> buckets(5);
            for (const StoredResource* k : kids) {
                long long t;
                auto an = k->Annotations.find(kLastUsed);
                if (an == k->Annotations.end() || !parseRFC3339(an->second, &t)) t = k->CreationSeq;
                const std::string& st = k->obj.Status.State;
                auto dd = k->Annotations.find(kDeleteDevice);
                const bool del = dd != k->Annotations.end() && dd->second == "true";
                int b;
                if (st == "None" || (st == "Attaching" && k->obj.Status.DeviceID.empty())) b = 0;
                else if (st == "Online" && del) b = 1;
                else if (st == "Attaching") b = 2;
                else if (st == "Online") b = 3;
                else b = 4;
                buckets[(size_t)b].push_back({k->obj.Name, t});
            }
            for (auto& b : buckets)
                std::stable_sort(b.begin(), b.end(), [](const P& x, const P& y) { return x.key < y.key; });
            bool done = false;
            for (size_t i = 0; !done; ++i) {
                if (i >= buckets.size())   // Go: index out of range on resourcesByDeletionPriority[i]
                    return requeueOnErr(r, Error::New("runtime error: index out of range [5] with length 5"));
                for (const P& p : buckets[i]) {
                    r->Status.Resources.erase(p.name);
                    if (--resourcesToDelete == 0) { done = true; break; }
                }
            }
        }

        std::vector<std::string> allocatingNodes;
        const std::string& policy = r->Spec.AllocationPolicy;
        if (policy == "samenode" && !r->Spec.TargetNode.empty()) {   // :364-386
            if (!c_->getNode(r->Spec.TargetNode)) return requeueOnErr(r, Error::New("the target node does not existed"));
            if (r->Spec.HasOtherSpec) {
                bool ok = false;
                Error e = c_->CheckNodeCapacitySufficient(r->Spec.TargetNode, r->Spec.OtherSpec, &ok);
                if (!e.ok()) return requeueOnErr(r, e);
                if (!ok) return requeueOnErr(r, Error::New("TargetNode does not meet spec's requirements"));
            }
            for (long long i = 0; i < resourcesToAllocate; ++i) allocatingNodes.push_back(r->Spec.TargetNode);
        }
        if (policy == "samenode" && r->Spec.TargetNode.empty()) {   // :387-444
            if (!r->Status.Resources.empty()) {
                for (long long i = 0; i < resourcesToAllocate; ++i) allocatingNodes.push_back(targetNodeForSamePolicy);
            } else {
                for (const Node& node : c_->nodes_) {
                    if (r->Spec.HasOtherSpec) {
                        bool ok = false;
                        Error e = c_->CheckNodeCapacitySufficient(node.Name, r->Spec.OtherSpec, &ok);
                        if (!e.ok()) return requeueOnErr(r, e);
                        if (!ok) continue;
                    }
                    bool occupied = false;
                    for (const auto& kv : c_->requests_) {
                        const ComposabilityRequest& req = kv.second;
                        if (req.Name == r->Name) continue;
                        std::string targetNode;
                        if (req.Spec.AllocationPolicy == "samenode") {
                            if (req.Spec.TargetNode.empty()) {
                                if (!req.Status.Resources.empty()) targetNode = req.Status.Resources.begin()->second.NodeName;
                            } else {
                                targetNode = req.Spec.TargetNode;
                            }
                        }
                        if (targetNode == node.Name) { occupied = true; break; }
                    }
                    if (occupied) continue;
                    for (long long i = 0; i < resourcesToAllocate; ++i) allocatingNodes.push_back(node.Name);
                    break;
                }
                if ((long long)allocatingNodes.size() != resourcesToAllocate)
                    return requeueOnErr(r, Error::New("insufficient number of available nodes"));
            }
        }
        if (policy == "differentnode") {   // :445-466
            for (const Node& node : c_->nodes_) {
                if (r->Spec.HasOtherSpec) {
                    bool ok = false;
                    Error e = c_->CheckNodeCapacitySufficient(node.Name, r->Spec.OtherSpec, &ok);
                    if (!e.ok()) return requeueOnErr(r, e);
                    if (!ok) continue;
                }
                if (!contains(allocatingNodes, node.Name) && !allocatedNodesForDifferentPolicy.count(node.Name))
                    allocatingNodes.push_back(node.Name);
                if ((long long)allocatingNodes.size() == resourcesToAllocate) break;
            }
            if ((long long)allocatingNodes.size() != resourcesToAllocate)
                return requeueOnErr(r, Error::New("insufficient number of available nodes"));
        }
        for (const std::string& n : allocatingNodes) {   // :471-479
            ScalarResourceStatus s;
            s.NodeName = n;
            r->Status.Resources[c_->GenerateComposableResourceName(r->Spec.Type)] = s;
        }
        r->Status.State = "Updating";
        r->Status.Error = "";
        r->Status.ScalarResource = r->Spec;
        c_->updateRequest(*r);
        return Error::Nil();
    }

    Error handleUpdatingState(ComposabilityRequest* r, long long* requeue) {   // :487-560
        if (r->DeletionTimestampSet) {
            r->Status.State = "Cleaning";
            c_->updateRequest(*r);
            return Error::Nil();
        }
        if (!(r->Status.ScalarResource == r->Spec)) {
            r->Status.State = "NodeAllocating";
            r->Status.ScalarResource = r->Spec;
            c_->updateRequest(*r);
            return Error::Nil();
        }
        std::set<std::string> existed;
        std::vector<std::string> surplus;
        for (const StoredResource* k : children(r->Name, false)) {
            if (!r->Status.Resources.count(k->obj.Name)) surplus.push_back(k->obj.Name);
            else existed.insert(k->obj.Name);
        }
        for (const std::string& n : surplus) c_->deleteResource(n);
        for (const auto& kv : r->Status.Resources) {
            if (existed.count(kv.first)) continue;
            StoredResource s;
            s.obj.Name = kv.first;
            s.obj.Labels[kManagedBy] = r->Name;
            s.obj.Spec.Type = r->Spec.Type;
            s.obj.Spec.Model = r->Spec.Model;
            s.obj.Spec.TargetNode = kv.second.NodeName;
            s.obj.Spec.ForceDetach = r->Spec.ForceDetach;
            c_->createResource(s);
        }
        bool canRun = true;
        for (const auto& kv : r->Status.Resources)
            if (kv.second.State != "Online") canRun = false;
        if (canRun) {
            r->Status.State = "Running";
            r->Status.Error = "";
            r->Status.ScalarResource = r->Spec;
            c_->updateRequest(*r);
            return Error::Nil();
        }
        *requeue = 30;
        return Error::Nil();
    }

    Error handleRunningState(ComposabilityRequest* r, long long* requeue) {   // :562-586
        if (r->DeletionTimestampSet) {
            r->Status.State = "Cleaning";
            c_->updateRequest(*r);
            return Error::Nil();
        }
        if (!(r->Status.ScalarResource == r->Spec)) {
            r->Status.State = "NodeAllocating";
            r->Status.ScalarResource = r->Spec;
            c_->updateRequest(*r);
            return Error::Nil();
        }
        r->Status.Error = "";
        c_->updateRequest(*r);
        *requeue = 30;
        return Error::Nil();
    }

    Error handleCleaningState(ComposabilityRequest* r, long long* requeue) {   // :588-612
        const std::vector<const StoredResource*> kids = children(r->Name, false);
        if (kids.empty()) {
            r->Status.State = "Deleting";
            c_->updateRequest(*r);
            return Error::Nil();
        }
        std::vector<std::string> names;
        for (const StoredResource* k : kids) names.push_back(k->obj.Name);
        for (const std::string& n : names) c_->deleteResource(n);
        r->Status.Error = "";
        c_->updateRequest(*r);
        *requeue = 30;
        return Error::Nil();
    }

    Error handleDeletingState(ComposabilityRequest* r) {   // :614-625
        removeStr(&r->Finalizers, kFinalizer);
        c_->updateRequest(*r);
        return Error::Nil();
    }

    Cluster* c_;
};

// =====================================================================================
// ComposableResourceReconciler  (internal/controller/composableresource_controller.go)
// =====================================================================================
class SimProvider : public controller::CdiProvider {
public:
    explicit SimProvider(Cluster* c) : c_(c) {}
    // fake fabric: the device of node i is physical GPU (i mod n); CDIDeviceID res-<request>-<k>
    Error AddResource(const controller::ComposableResource& inst, std::string* dev, std::string* cdi) override {
        size_t idx = 0;
        for (size_t i = 0; i < c_->nodes_.size(); ++i)
            if (c_->nodes_[i].Name == inst.Spec.TargetNode) idx = i;
        *dev = c_->uuids_[idx % c_->uuids_.size()];
        auto mb = inst.Labels.find(kManagedBy);
        const std::string owner = mb == inst.Labels.end() ? std::string("orphan") : mb->second;
        *cdi = "res-" + owner + "-" + std::to_string(c_->cdi_serial_[owner]++);
        c_->attached_.insert(inst.Name);
        return Error::Nil();
    }
    Error RemoveResource(controller::ComposableResource& inst) override {
        c_->attached_.erase(inst.Name);
        return Error::Nil();
    }

private:
    Cluster* c_;
};

class SimNodeOps : public controller::NodeOps {
public:
    explicit SimNodeOps(Cluster* c) : c_(c) {}
    Error CheckNoGPULoads(const std::string&) override { return Error::Nil(); }
    Error RestartDaemonset(const std::string&, const std::string&) override { return Error::Nil(); }
    Error RunNvidiaSmi(const std::string&) override { return Error::Nil(); }
    Error CheckGPUVisible(const std::string&, const controller::ComposableResource& r, bool* visible) override {
        *visible = false;
        if (!c_->attached_.count(r.Name)) return Error::Nil();   // logically detached
        bool listed = false;
        for (const std::string& u : c_->uuids_)
            if (u == r.Status.DeviceID) listed = true;           // internal/utils/gpus.go:78-82
        if (!listed) return Error::Nil();
        if (c_->probe_) {
            int idx = -1;
            for (size_t i = 0; i < c_->ctx_->devs.size(); ++i)
                if (std::string(c_->ctx_->devs[i]->info.gpu_uuid, strnlen(c_->ctx_->devs[i]->info.gpu_uuid, 48)) ==
                    r.Status.DeviceID)
                    idx = (int)i;
            if (idx < 0) return Error::Nil();
            // Non-blocking reconcile: the first pass begins the probe on the device's stream and
            // asks for a requeue; a later pass collects it.  One reconcile worker therefore keeps
            // every GPU of the box busy (a device serves one attach at a time, in arrival order).
            std::deque<std::string>& owners = c_->probe_owner_[idx];
            size_t pos = 0;
            while (pos < owners.size() && owners[pos] != r.Name) ++pos;
            if (pos == owners.size()) {       // not probing yet
                if (owners.size() < 2) {      // a free lane: enqueue behind whatever is running on the device
                    if (ctx_probe_begin(c_->ctx_, idx) != CRO_OK) {
                        if (owners.empty()) c_->probe_owner_.erase(idx);
                        return Error::New("cuda probe failed: could not start the probe");
                    }
                    if (!owners.empty() && idx < 16) ++c_->stats.gpu[idx].begins_behind_running;
                    owners.push_back(r.Name);
                    c_->traceEvent('b', idx);
                } else if (c_->probe_waiting_.insert(r.Name).second) {
                    c_->dev_waiters_[idx].push_back(r.Name);   // both lanes taken: queue behind them
                    c_->traceEvent('w', idx);
                }
                probePending = true;
                return Error::Nil();
            }
            if (pos > 0) {                    // ours is the second in line: results come out oldest first
                probePending = true;
                return Error::Nil();
            }
            if (!ctx_probe_poll(c_->ctx_, idx)) {   // ours, still running
                c_->probe_notified_.erase(idx);
                probePending = true;
                return Error::Nil();
            }
            cro_probe_result pr;
            ++c_->stats.probes;
            int rc = ctx_probe_end(c_->ctx_, idx, &pr);
            c_->traceEvent('c', idx);
            if (rc == CRO_OK && idx < 16) {   // how busy the reconcile worker kept this GPU (the device's own %globaltimer)
                Stats::Gpu& g = c_->stats.gpu[idx];
                if (g.probes++ == 0) g.first_start_ns = pr.t_start_ns;
                else if (pr.t_start_ns > g.last_end_ns) {          // the device sat idle between two probes for this long
                    const unsigned long long gap = pr.t_start_ns - g.last_end_ns;
                    g.gap_ns += gap;
                    g.max_gap_ns = std::max(g.max_gap_ns, gap);
                    if (gap > 100000) ++g.gaps_over_100us;
                }
                g.busy_ns += pr.total_ns;
                g.last_end_ns = pr.t_start_ns + pr.total_ns;
            }
            c_->releaseDevice(idx);
            if (rc != CRO_OK) {
                ++c_->stats.probe_failures;
                return Error::New(std::string("cuda probe failed: ") + cro_strerror(rc));
            }
        }
        *visible = true;
        return Error::Nil();
    }
    bool probePending = false;   // set when CheckGPUVisible is waiting on a probe rather than on the cluster

private:
    Cluster* c_;
};

class ResourceReconciler {
public:
    explicit ResourceReconciler(Cluster* c) : c_(c), provider_(c), node_(c) {}

    Error Reconcile(const std::string& key, long long* requeue) {   // :73-126
        *requeue = 0;
        auto it = c_->resources_.find(key);
        if (it == c_->resources_.end()) return Error::Nil();   // NotFound: do not requeue
        StoredResource s = it->second;
        controller::ComposableResource& res = s.obj;

        // performGarbageCollection :128-174
        if (!res.Spec.TargetNode.empty() && !c_->getNode(res.Spec.TargetNode)) {
            bool needRet = false;
            if (res.Status.State != "Deleting") {
                res.Status.State = "Deleting";
                res.Status.Error = "target node " + res.Spec.TargetNode + " not found";
                c_->updateResource(s);
                needRet = true;
            }
            if (!res.DeletionTimestampSet) {
                c_->deleteResource(res.Name);
                needRet = true;
            }
            if (needRet) return Error::Nil();
        }
        if (c_->deviceResourceType_ != "DEVICE_PLUGIN" && c_->deviceResourceType_ != "DRA") {   // adapter :42-45
            Error e = Error::New("the env variable DEVICE_RESOURCE_TYPE has an invalid value: '" + c_->deviceResourceType_ + "'");
            res.Status.Error = e.msg;
            c_->updateResource(s);
            return e;
        }

        controller::ComposableResourceReconciler rec(&provider_, &node_);
        controller::Result result;
        Error err;
        const std::string st = res.Status.State;
        if (st.empty()) {
            if (!contains(s.Finalizers, kFinalizer)) s.Finalizers.push_back(kFinalizer);   // :179-184
            err = rec.handleNoneState(&res, &result);
        } else if (st == "Attaching") {
            err = rec.handleAttachingState(&res, c_->deviceResourceType_, &result);
        } else if (st == "Online") {
            err = rec.handleOnlineState(&res, &result);
            if (res.DeleteRequested) {   // r.Delete(resource) on itself (:298)
                res.DeleteRequested = false;
                c_->deleteResource(res.Name);
                res.DeletionTimestampSet = true;
            }
        } else if (st == "Detaching") {
            err = rec.handleDetachingState(&res, c_->deviceResourceType_, &result);
        } else if (st == "Deleting") {
            removeStr(&s.Finalizers, kFinalizer);   // :409-421
        }
        // every intermediate Status().Update the reference issues would have produced the same final
        // object; persist once (the count of updates is what the stats report)
        c_->stats.status_updates += rec.statusUpdates.empty() ? 0 : (long long)rec.statusUpdates.size() - 1;
        c_->updateResource(s);
        *requeue = node_.probePending ? -1 : result.RequeueAfterSeconds;
        return err;
    }

private:
    Cluster* c_;
    SimProvider provider_;
    SimNodeOps node_;
};

// A failed write ends the handler where it stands (Go: `if err := r.Update(...); err != nil { return requeueOnErr }`)
// and the reconcile returns that error; nothing the handler did after the last good write survives.
Error Cluster::reconcileRequest(const std::string& key, long long* requeue) {
    RequestReconciler r(this);
    try {
        return r.Reconcile(key, requeue);
    } catch (const ApiFault& f) {
        *requeue = 0;
        return Error::New(f.msg);
    }
}
Error Cluster::reconcileResource(const std::string& key, long long* requeue) {
    ResourceReconciler r(this);
    try {
        return r.Reconcile(key, requeue);
    } catch (const ApiFault& f) {
        *requeue = 0;
        return Error::New(f.msg);
    }
}

Error Cluster::ReconcileRequestOnce(const std::string& name) {
    long long rq = 0;
    ++stats.request_reconciles;
    return reconcileRequest(name, &rq);
}

// Requeues the attaches whose probe has finished (called between reconciles), and drops the
// ownership of devices whose attach disappeared meanwhile.
void Cluster::pollProbes(bool block) {
    if (probe_owner_.empty()) return;
    std::vector<int> orphaned;
    bool woke = false;
    for (const auto& kv : probe_owner_) {
        if (kv.second.empty()) continue;
        auto it = resources_.find(kv.second.front());
        if (it == resources_.end() || it->second.obj.Status.State != "Attaching") {
            orphaned.push_back(kv.first);
        } else if (!probe_notified_.count(kv.first) && ctx_probe_poll(ctx_, kv.first)) {
            probe_notified_.insert(kv.first);
            enqueueResourceFront(kv.second.front());   // its owner can collect now
            woke = true;
        }
    }
    for (int dev : orphaned) {   // the attach vanished: discard its probe, hand the device on
        cro_probe_result discard;
        ctx_probe_end(ctx_, dev, &discard);
        releaseDevice(dev);
        woke = true;
    }
    if (!woke && block && !probe_owner_.empty()) {
        // nothing else to reconcile: wait for WHICHEVER device finishes first (blocking on one
        // particular stream would leave the others idle once they drift apart)
        bool any_unnotified = false;
        for (const auto& kv : probe_owner_) any_unnotified |= !kv.second.empty() && !probe_notified_.count(kv.first);
        while (any_unnotified && !woke) {
            for (const auto& kv : probe_owner_) {
                if (kv.second.empty() || probe_notified_.count(kv.first) || !ctx_probe_poll(ctx_, kv.first)) continue;
                probe_notified_.insert(kv.first);
                enqueueResourceFront(kv.second.front());
                woke = true;
            }
            if (!woke) usleep(20);
        }
    }
}

// The attach that owned `dev` is done with it: the next one queued behind it gets a turn.
void Cluster::releaseDevice(int dev) {
    auto own = probe_owner_.find(dev);
    if (own != probe_owner_.end()) {
        if (!own->second.empty()) own->second.pop_front();       // the oldest probe has been collected
        if (own->second.empty()) probe_owner_.erase(own);
    }
    probe_notified_.erase(dev);
    auto q = dev_waiters_.find(dev);
    if (q == dev_waiters_.end()) return;
    while (!q->second.empty()) {
        const std::string next = q->second.front();
        q->second.pop_front();
        probe_waiting_.erase(next);
        if (resources_.count(next)) {
            enqueueResourceFront(next);
            break;
        }
    }
}

// =====================================================================================
// UpstreamSyncer  (internal/controller/upstreamsyncer_controller.go:77-159)
// =====================================================================================
// devices: what CdiProvider.GetResources() returned ([]cdi.DeviceInfo, internal/cdi/client.go:25-32) —
// or, on a node-local agent, the gathered probe results: a device the node can enumerate and probe
// but no ComposableResource owns is exactly the drift this loop repairs.
Error Cluster::SyncUpstream(const gojson::Value& devices, long long now_s) {
    if (devices.kind != gojson::Value::Array) return Error::New("failed to fetch data from upstream server: not a device list");
    std::set<std::string> existingDeviceIDs;                                   // :88-93
    for (const auto& kv : resources_)
        if (!kv.second.obj.Status.DeviceID.empty()) existingDeviceIDs.insert(kv.second.obj.Status.DeviceID);
    std::set<std::string> upstream;
    for (const auto& d : devices.arr) {                                        // :95-121
        const std::string deviceID = d->get_string("device_id");
        upstream.insert(deviceID);
        if (existingDeviceIDs.count(deviceID)) {
            missing_devices_.erase(deviceID);
            continue;
        }
        auto it = missing_devices_.find(deviceID);
        if (it == missing_devices_.end()) {
            missing_devices_[deviceID] = now_s;                                // start tracking
        } else if (now_s - it->second > 10 * 60) {                             // missingDeviceGracePeriod :37
            // createDetachCR :138-159.  GenerateName is a full "gpu-<uuid4>", so the API server
            // appends 5 more characters (SURVEY.md Appendix A-10).
            StoredResource s;
            static const char alnum[] = "bcdfghjklmnpqrstvwxz2456789";
            std::string name = GenerateComposableResourceName("gpu");
            for (int k = 0; k < 5; ++k) name.push_back(alnum[rng_() % (sizeof alnum - 1)]);
            s.obj.Name = name;
            s.obj.Labels["cohdi.io/ready-to-detach-device-id"] = deviceID;
            s.obj.Labels["cohdi.io/ready-to-detach-cdi-device-id"] = d->get_string("cdi_device_id");
            s.obj.Spec.Type = d->get_string("device_type");
            s.obj.Spec.Model = d->get_string("model");
            s.obj.Spec.TargetNode = d->get_string("node_name");
            s.obj.Spec.ForceDetach = false;
            attached_.insert(name);   // the device IS on the node: that is the premise of the repair
            createResource(s);
            missing_devices_.erase(deviceID);
        }
    }
    for (auto it = missing_devices_.begin(); it != missing_devices_.end();)   // :123-133
        it = upstream.count(it->first) ? std::next(it) : missing_devices_.erase(it);
    return Error::Nil();
}

Error Cluster::ReconcileResourceOnce(const std::string& name) {
    long long rq = 0;
    ++stats.resource_reconciles;
    return reconcileResource(name, &rq);
}

// ---- event loop ----------------------------------------------------------------------
void Cluster::Run(long long max_reconciles) {
    using clk = std::chrono::steady_clock;
    const auto t0 = clk::now();
    long long n = 0;
    long long changes_at_flush = -1;
    for (;;) {
        while ((!req_queue_.empty() || !res_queue_.empty()) && n < max_reconciles) {
            // Look for finished probes every 100 us of reconciling.  (Round 1 polled when n % 4 == 0 — but n advances
            // by two per turn while both queues hold work, so an odd n never hit a multiple of four again and finished
            // probes sat uncollected until a queue drained: a hole per GPU at the start of a storm.)
            const auto now_poll = clk::now();
            if (now_poll - last_poll_ >= std::chrono::microseconds(100)) {
                last_poll_ = now_poll;
                pollProbes(false);
            }
            // one worker per controller (MaxConcurrentReconciles default 1), interleaved
            if (!res_queue_.empty()) {
                const std::string key = res_queue_.front();
                res_queue_.pop_front();
                res_queued_.erase(key);
                long long rq = 0;
                const auto a = clk::now();
                Error e = reconcileResource(key, &rq);
                stats.reconcile_ns.push_back(std::chrono::duration_cast<std::chrono::nanoseconds>(clk::now() - a).count());
                ++stats.resource_reconciles;
                ++n;
                if (!e.ok()) { ++stats.reconcile_errors; res_timers_.insert(key); }   // back-off requeue
                else if (rq < 0) { /* parked on a GPU (owner or queued behind one): pollProbes wakes it */ }
                else if (rq > 0) res_timers_.insert(key);
            }
            if (!req_queue_.empty()) {
                const std::string key = req_queue_.front();
                req_queue_.pop_front();
                req_queued_.erase(key);
                long long rq = 0;
                const auto a = clk::now();
                Error e = reconcileRequest(key, &rq);
                stats.reconcile_ns.push_back(std::chrono::duration_cast<std::chrono::nanoseconds>(clk::now() - a).count());
                ++stats.request_reconciles;
                ++n;
                if (!e.ok()) { ++stats.reconcile_errors; req_timers_.insert(key); }
                else if (rq > 0) req_timers_.insert(key);
            }
        }
        if (n >= max_reconciles) break;
        if (!probe_owner_.empty()) {   // nothing else to do: wait for the next probe to finish
            const auto b0 = clk::now();
            pollProbes(true);
            stats.blocked_ns += std::chrono::duration_cast<std::chrono::nanoseconds>(clk::now() - b0).count();
            continue;
        }
        // queue drained: fire the RequeueAfter timers, unless the last round changed nothing
        if ((req_timers_.empty() && res_timers_.empty()) || changes_ == changes_at_flush) break;
        changes_at_flush = changes_;
        ++stats.timer_rounds;
        for (const std::string& k : req_timers_) enqueueRequest(k);
        for (const std::string& k : res_timers_) enqueueResource(k);
        req_timers_.clear();
        res_timers_.clear();
    }
    stats.wall_s += std::chrono::duration<double>(clk::now() - t0).count();
}

std::string Cluster::DumpJSON() const {
    gojson::Writer w;
    w.begin_object();
    w.key("requests").begin_object();
    for (const auto& kv : requests_) {
        w.key(kv.first.c_str()).begin_object();
        w.key("spec").raw(kv.second.Spec.MarshalJSON());
        w.key("status").raw(kv.second.Status.MarshalJSON());
        w.field("deleting", kv.second.DeletionTimestampSet);
        w.key("finalizers").begin_array();
        for (const auto& f : kv.second.Finalizers) w.value(f);
        w.end_array();
        w.end_object();
    }
    w.end_object();
    w.key("missing_devices").begin_object();
    for (const auto& kv : missing_devices_) w.key(kv.first.c_str()).value(kv.second);
    w.end_object();
    w.key("resources").begin_object();
    for (const auto& kv : resources_) {
        const controller::ComposableResource& r = kv.second.obj;
        w.key(kv.first.c_str()).begin_object();
        w.key("spec").begin_object().field("type", r.Spec.Type).field("model", r.Spec.Model).field("target_node", r.Spec.TargetNode);
        w.field_omitempty("force_detach", r.Spec.ForceDetach).end_object();
        w.key("status").raw(r.Status.MarshalJSON());
        w.key("labels").string_map(r.Labels);
        w.field("deleting", r.DeletionTimestampSet);
        w.key("finalizers").begin_array();
        for (const auto& f : kv.second.Finalizers) w.value(f);
        w.end_array();
        w.end_object();
    }
    w.end_object();
    w.end_object();
    return w.take();
}

std::string Cluster::StatsJSON() const {
    std::vector<long long> v = stats.reconcile_ns;
    std::sort(v.begin(), v.end());
    auto pct = [&](double p) -> long long { return v.empty() ? 0 : v[std::min(v.size() - 1, (size_t)(p * (double)v.size()))]; };
    long long running = 0, online = 0;
    for (const auto& kv : requests_) running += kv.second.Status.State == "Running";
    for (const auto& kv : resources_) online += kv.second.obj.Status.State == "Online";
    gojson::Writer w;
    w.begin_object();
    w.field("requests", (long long)requests_.size()).field("requests_running", running);
    w.field("resources", (long long)resources_.size()).field("resources_online", online);
    w.field("request_reconciles", stats.request_reconciles).field("resource_reconciles", stats.resource_reconciles);
    w.field("status_updates", stats.status_updates).field("spec_bytes", stats.spec_bytes);
    w.field("probes", stats.probes).field("probe_failures", stats.probe_failures);
    w.field("reconcile_errors", stats.reconcile_errors).field("timer_rounds", stats.timer_rounds);
    w.field("reconcile_p50_ns", pct(0.50)).field("reconcile_p99_ns", pct(0.99));
    w.field("wall_us", (long long)(stats.wall_s * 1e6));
    long long total_ns = 0, max_ns = 0;
    for (long long x : stats.reconcile_ns) { total_ns += x; max_ns = std::max(max_ns, x); }
    w.field("reconcile_total_us", total_ns / 1000).field("reconcile_max_us", max_ns / 1000).field("worker_blocked_us", stats.blocked_ns / 1000);
    if (stats.tracing) {
        w.key("trace").begin_array();
        for (const Stats::Ev& e : stats.trace) {
            w.begin_array();
            w.value((long long)e.t_us).value(std::string(1, e.what)).value((long long)e.dev);
            w.end_array();
        }
        w.end_array();
    }
    w.key("gpus").begin_array();
    for (const Stats::Gpu& g : stats.gpu) {
        if (!g.probes) continue;
        w.begin_object();
        w.field("probes", g.probes).field("busy_us", (long long)(g.busy_ns / 1000));
        w.field("span_us", (long long)((g.last_end_ns - g.first_start_ns) / 1000));
        w.field("idle_between_probes_us", (long long)(g.gap_ns / 1000)).field("max_gap_us", (long long)(g.max_gap_ns / 1000));
        w.field("gaps_over_100us", g.gaps_over_100us).field("begins_behind_running", g.begins_behind_running);
        w.end_object();
    }
    w.end_array();
    w.field("timers", std::string("RequeueAfter fires when the queue drains; stops when a round changes nothing"));
    w.end_object();
    return w.take();
}

}  // namespace sim
}  // namespace cro
