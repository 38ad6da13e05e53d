// deepterrainrl_b200 -- scene assembly from the reference's own files (see ref_loader.h).
#include "ref_loader.h"

#include <cmath>

namespace trl {

namespace {

const char* kCharNames[] = {"none", "dog", "raptor"};
const char* kCtrlNames[] = {"none", "dog", "dog_cacla", "dog_mace", "goat_mace", "raptor", "raptor_cacla", "raptor_mace"};
const char* kTerrainTypes[] = {"flat", "gaps", "steps", "walls", "bumps", "mixed", "narrow_gaps", "slopes", "slopes_gaps",
                               "slopes_walls", "slopes_steps", "slopes_mixed", "slopes_narrow_gaps", "cliffs"};
struct ParamDef { const char* name; double dflt; };
// cTerrainGen2D::gParamDefs (sim/TerrainGen2D.cpp:8-56)
const ParamDef kTerrainParams[40] = {
    {"GapSpacingMin", 4}, {"GapSpacingMax", 7}, {"GapWMin", 0.5}, {"GapWMax", 2}, {"GapHMin", -2}, {"GapHMax", -2},
    {"WallSpacingMin", 6}, {"WallSpacingMax", 8}, {"WallWMin", 0.2}, {"WallWMax", 0.2}, {"WallHMin", 0.25}, {"WallHMax", 0.5},
    {"StepSpacingMin", 5}, {"StepSpacingMax", 7}, {"StepH0Min", 0.1}, {"StepH0Max", 0.4}, {"StepH1Min", -0.4}, {"StepH1Max", -0.1},
    {"BumpHMin", 0}, {"BumpHMax", 0.03},
    {"NarrowGapSpacingMin", 3}, {"NarrowGapSpacingMax", 6}, {"NarrowGapDistMin", 0.1}, {"NarrowGapDistMax", 0.4},
    {"NarrowGapWMin", 0.15}, {"NarrowGapWMax", 0.5}, {"NarrowGapDepthMin", -2}, {"NarrowGapDepthMax", -2},
    {"NarrowGapCountMin", 1}, {"NarrowGapCountMax", 4},
    {"CliffSpacingMin", 5}, {"CliffSpacingMax", 7}, {"CliffH0Min", 0.1}, {"CliffH0Max", 0.4}, {"CliffH1Min", -0.4},
    {"CliffH1Max", -0.1}, {"CliffMiniCountMax", 0},
    {"SlopeDeltaRange", 0.25}, {"SlopeDeltaMin", -0.35}, {"SlopeDeltaMax", 0.35}};
const char* kNetLayerNames[13] = {"terr_conv0", "terr_conv1", "terr_conv2", "terr_ip0", "ip0", "val_ip0", "val_ip1",
                                  "a0_ip0", "a0_ip1", "a1_ip0", "a1_ip1", "a2_ip0", "a2_ip1"};

template <size_t N>
int index_of(const char* const (&names)[N], const std::string& v, const char* what) {
    for (size_t i = 0; i < N; ++i) if (v == names[i]) return (int)i;
    throw std::runtime_error(std::string("unknown ") + what + ": " + v);
}

std::string join(const std::string& root, const std::string& rel) {
    if (!rel.empty() && rel[0] == '/') return rel;
    return root.empty() ? rel : root + "/" + rel;
}

// one gait-controller file -> flat parameter vector (sim/DogController.cpp:470-523, sim/RaptorController.cpp ReadParams)
std::vector<double> read_ctrl_params(const std::string& path, bool raptor) {
    static const char* dog_misc[] = {"TransTime", "Cv", "BackForceX", "BackForceY", "FrontForceX", "FrontForceY"};
    static const char* dog_states[] = {"BackStance", "Extend", "FrontStance", "Gather"};
    static const char* dog_sp[] = {"SpineCurve", "Shoulder", "Elbow", "Hip", "Knee", "Ankle"};
    static const char* rap_misc[] = {"TransTime", "Cv", "Cd", "ForceX", "ForceY"};
    static const char* rap_states[] = {"Contact", "Down", "Passing", "Up"};
    static const char* rap_sp[] = {"RootPitch", "SpineCurve", "StanceHip", "StanceKnee", "StanceAnkle", "SwingHip", "SwingKnee", "SwingAnkle"};
    JValue d = load_json(path);
    const JValue* misc = d.get("MiscParams");
    const JValue* sp = d.get("StateParams");
    if (!misc || !sp) throw std::runtime_error("controller file without MiscParams / StateParams: " + path);
    std::vector<double> v;
    const int nm = raptor ? 5 : 6, ns = raptor ? 8 : 6;
    for (int i = 0; i < nm; ++i) v.push_back(misc->number(raptor ? rap_misc[i] : dog_misc[i], 0.0));
    for (int s = 0; s < 4; ++s) {
        const JValue* st = sp->get(raptor ? rap_states[s] : dog_states[s]);
        if (!st) throw std::runtime_error("controller file misses a state block: " + path);
        for (int j = 0; j < ns; ++j) v.push_back(st->number(raptor ? rap_sp[j] : dog_sp[j], 0.0));
    }
    return v;
}

}  // namespace

TerrainFile read_terrain_file(const std::string& path) {
    TerrainFile tf;
    JValue t = load_json(path);
    std::string type = t.string("Type", "flat");
    if (type.empty()) type = "flat";
    tf.type = index_of(kTerrainTypes, type, "terrain type");
    if (const JValue* ps = t.get("Params"))
        for (const JValue& s : ps->arr) {
            for (int i = 0; i < 40; ++i) tf.params.push_back(s.number(kTerrainParams[i].name, kTerrainParams[i].dflt));
            ++tf.n_sets;
        }
    return tf;
}

std::string join_path(const std::string& root, const std::string& rel) { return join(root, rel); }

CharacterRecords read_character_file(const std::string& path, const std::string& root, bool raptor, int expect_nj) {
    JValue ch = load_json(path);
    const JValue* skel = ch.get("Skeleton");
    const JValue* joints = skel ? skel->get("Joints") : nullptr;
    const JValue* bodies = ch.get("BodyDefs");
    const JValue* pds = ch.get("PDControllers");
    const JValue* ctrls = ch.get("Controllers");
    if (!joints || !bodies || !pds || !ctrls) throw std::runtime_error("character file misses Skeleton / BodyDefs / PDControllers / Controllers");
    CharacterRecords cr;
    const int nj = (int)joints->arr.size();
    if (expect_nj >= 0 && nj != expect_nj)
        throw std::runtime_error("the character's topology differs from the scene's: " + std::to_string(nj) + " joints, the scene's character has " +
                                 std::to_string(expect_nj));
    if (bodies->arr.size() < (size_t)nj || pds->arr.size() < (size_t)nj)
        throw std::runtime_error("character file has fewer BodyDefs / PDControllers than joints");
    cr.nj = nj;
    std::vector<double>&J = cr.joints, &B = cr.bodies, &P = cr.pd;
    J.assign(7 * nj, 0.0); B.assign(9 * nj, 0.0); P.assign(6 * nj, 0.0);
    int ndof = 0;
    for (int i = 0; i < nj; ++i) {
        const JValue& j = joints->arr[i];
        double* r = &J[7 * i];
        r[0] = j.number("Type", 0); r[1] = j.number("Parent", -1); r[2] = j.number("AttachX", 0); r[3] = j.number("AttachY", 0);
        r[4] = j.number("AttachZ", 0); r[5] = j.number("LimLow", 1); r[6] = j.number("LimHigh", 0);
        const int type = (int)r[0];
        const bool is_root = r[1] < 0;
        ndof += (type == 1) ? 3 : ((type == 3) ? (is_root ? 3 : 0) : 1);   // cKinTree::GetParamSize (anim/KinTree.cpp:731-757)
        const JValue& b = bodies->arr[i];
        const std::string shape = b.string("Shape", "null");
        double* q = &B[9 * i];
        q[0] = shape == "box" ? 0 : (shape == "capsule" ? 1 : -1);
        q[1] = b.number("Mass", 0); q[2] = b.number("AttachX", 0); q[3] = b.number("AttachY", 0); q[4] = b.number("AttachZ", 0);
        q[5] = b.number("Theta", 0); q[6] = b.number("Param0", 0); q[7] = b.number("Param1", 0); q[8] = b.number("Param2", 0);
        const JValue& p = pds->arr[i];
        double* w = &P[6 * i];
        w[0] = p.number("Kp", 0); w[1] = p.number("Kd", 0); w[2] = p.number("TorqueLim", 0); w[3] = p.number("TargetTheta", 0);
        w[4] = p.number("TargetVel", 0); w[5] = p.number("UseWorldCoord", 0);
    }
    if (nj > 0) J[2] = J[3] = J[4] = 0.0;   // PostProcessJointMat zeroes the root attach point (anim/KinTree.cpp:1004-1016)
    cr.ndof = ndof;

    const JValue* files = ctrls->get("Files");
    const JValue* actions = ctrls->get("Actions");
    if (files) for (const JValue& f : files->arr) {
        std::vector<double> v = read_ctrl_params(join(root, f.str), raptor);
        cr.ctrl_params.insert(cr.ctrl_params.end(), v.begin(), v.end());
        ++cr.n_ctrl;
    }
    if (actions) for (const JValue& a : actions->arr) {
        for (const char* k : {"ParamIdx0", "ParamIdx1", "Blend", "Cyclic"}) cr.actions.push_back(a.number(k, 0));
        ++cr.n_actions;
    }
    cr.default_action = (int)ctrls->number("DefaultAction", 0);
    cr.grav_comp = ctrls->number("EnableGravityCompensation", 1) != 0 ? 1 : 0;
    cr.virt_forces = ctrls->number("EnableVirtualForces", 1) != 0 ? 1 : 0;
    return cr;
}

void build_scene_from_args(int argc, const char* const* argv, const std::string& root, ScenePack* out) {
    // CLI tokens first, then the arg file's, so the CLI wins on first-match lookup (optimizer/Main.cpp:19-32)
    ArgList args;
    args.append_args(argc, argv);
    std::string arg_file;
    if (args.find("arg_file", &arg_file)) args.append_file(join(root, arg_file));

    const std::string char_file = args.str("character_file", "");
    if (char_file.empty()) throw std::runtime_error("No character file specified.");
    const int char_type = index_of(kCharNames, args.str("char_type", "none"), "char_type");
    const int ctrl = index_of(kCtrlNames, args.str("char_ctrl", "none"), "char_ctrl");
    const bool raptor = char_type == 2;
    const CharacterRecords cr = read_character_file(join(root, char_file), root, raptor);
    const int nj = cr.nj, ndof = cr.ndof, n_ctrl = cr.n_ctrl, n_actions = cr.n_actions;
    const int default_action = cr.default_action, grav_comp = cr.grav_comp, virt_forces = cr.virt_forces;
    const std::vector<double>&J = cr.joints, &B = cr.bodies, &P = cr.pd, &C = cr.ctrl_params, &A = cr.actions;

    std::vector<double> pose0(ndof, 0.0), vel0(ndof, 0.0);
    const std::string state_file = args.str("state_file", "");
    if (!state_file.empty()) {
        JValue st = load_json(join(root, state_file));
        const JValue* pp = st.get("Pose");
        const JValue* vv = st.get("Vel");
        if (!pp || !vv || (int)pp->arr.size() != ndof || (int)vv->arr.size() != ndof) throw std::runtime_error("state file does not match the character's dof count");
        for (int k = 0; k < ndof; ++k) { pose0[k] = pp->arr[k].num; vel0[k] = vv->arr[k].num; }
    }

    std::vector<double> tdefault(40);
    for (int i = 0; i < 40; ++i) tdefault[i] = kTerrainParams[i].dflt;
    const std::string terrain_file = args.str("terrain_file", "");
    TerrainFile tf;
    if (!terrain_file.empty()) tf = read_terrain_file(join(root, terrain_file));
    const int terrain_type = tf.type, n_sets = tf.n_sets;
    const std::vector<double>& tparams = tf.params;

    const bool has_init_x = args.has("char_init_pos_x");
    const std::string model = args.str("policy_model", "");
    const int has_net = (!args.str("policy_net", "").empty() && !model.empty()) ? 1 : 0;

    out->set_i32("meta_i32", {char_type, ctrl, (int)args.num("num_update_steps", 20), (int)args.num("num_sim_substeps", 1), has_init_x ? 1 : 0,
                              terrain_type, n_sets, has_net, nj, ndof, n_ctrl, n_actions, default_action, grav_comp, virt_forces,
                              (int)args.num("tuple_buffer_size", 16)});
    out->set_f64("meta_f64", {0.0, -9.8, args.num("char_init_pos_x", 0.0), args.num("terrain_blend", 0.0), args.num("exp_rate", 0.1),
                              args.num("exp_temp", 1.0), args.num("exp_base_rate", 0.01), args.num("world_scale", 1.0)});
    out->set_f64("joints", J); out->set_f64("bodies", B); out->set_f64("pd", P); out->set_f64("ctrl_params", C); out->set_f64("actions", A);
    out->set_f64("pose0", pose0); out->set_f64("vel0", vel0); out->set_f64("terrain_params", tparams); out->set_f64("terrain_default_params", tdefault);

    if (has_net) {
        H5Reader h5(join(root, model));
        int frag = 0;
        for (const char* layer : kNetLayerNames) {
            for (int k = 0; k < 2; ++k) {
                auto it = h5.datasets().find(std::string("/data/") + layer + "/" + std::to_string(k));
                if (it == h5.datasets().end()) throw std::runtime_error(std::string("model file misses layer ") + layer);
                out->set_f64(std::string("net_") + layer + (k == 0 ? "_w" : "_b"), it->second);
                if (std::string(layer) == "a0_ip1" && k == 1) frag = (int)it->second.size();
            }
        }
        std::string scale_path = join(root, model);
        size_t dot = scale_path.rfind('.');
        scale_path = scale_path.substr(0, dot) + "_scale.txt";   // cNeuralNet::GetOffsetScaleFile (learning/NeuralNet.cpp:1174-1180)
        JValue sc = load_json(scale_path);
        const char* keys[4] = {"InputOffset", "InputScale", "OutputOffset", "OutputScale"};
        const char* names[4] = {"net_in_offset", "net_in_scale", "net_out_offset", "net_out_scale"};
        size_t n_in = 0, n_out = 0;
        for (int k = 0; k < 4; ++k) {
            const JValue* v = sc.get(keys[k]);
            if (!v) throw std::runtime_error(std::string("scale file misses ") + keys[k]);
            std::vector<double> vec;
            for (const JValue& x : v->arr) vec.push_back(x.num);
            if (k == 0) n_in = vec.size();
            if (k == 2) n_out = vec.size();
            out->set_f64(names[k], vec);
        }
        out->set_i32("net_dims", {(int)n_in, (int)n_in - 200, (int)n_out, (int)(n_out / (size_t)(frag + 1)), frag});
    }
}

}  // namespace trl
