// TEST INFRASTRUCTURE — not product code.  The animator binding (AnimatorsB200, lumixengine_b200/host/animation_b200.inl) over real
// Lumix::Model / Lumix::Animation / Lumix::Pose objects and scripted blend stacks, next to the reference's own evalBlendStack.  Built (through
// ref_root_motion_harness.cpp) into oracle/_ref/libanimation_shim_b200.so by oracle/build_ref.py, which cuts getPose .. evalBlendStack (controller.cpp) and the
// RuntimeContext constructor (nodes.cpp) out of the reference at build time into the overlay this file includes them from.
//   ref_pose_stack:      Model::getRelativePose + evalBlendStack + Pose::computeAbsolute on one scripted stack (tests/golden/stack_kat.npz)
//   ashim_run_animators: per frame, side A runs updateAnimator's :623-627 for every animator, side B runs AnimatorsB200::update and the
//                        same reference code for its referencePath()
#include "ref_anim_models_harness.cpp"

#define private public
#include "animation/controller.h"
#undef private
#include "core/stream.h"

#include "animators_b200.inl"

namespace Lumix::anim {
#include "animation/extracted_runtime_context.inl"
} // namespace Lumix::anim
namespace Lumix::anim {
#include "animation/extracted_blend_stack.inl"
} // namespace Lumix::anim

namespace {

// DefaultAllocator's destructor releases its small-allocation region with os::memRelease, which ref_stubs.cpp implements as munmap.  An
// allocator that never made a small allocation has no region, so at exit it would munmap(nullptr, 128 MB) and unmap whatever the process
// has mapped there.  log.cpp's logger creates the global allocator when this library loads; one small allocation here gives it its region.
const bool g_global_allocator_reserved = [] {
	IAllocator& a = getGlobalAllocator();
	a.deallocate(a.allocate(8, 8));
	return true;
}();

// the Controller the stacks refer to: zero storage with the members getPose / evalIK read (m_bone_masks, the path)
struct Controllers {
	explicit Controllers(IAllocator& allocator) {
		RawStorage<anim::Controller>* both[] = {&plain, &masked};
		for (RawStorage<anim::Controller>* m : both) {
			new (&m->get()->m_bone_masks) Array<BoneMask>(allocator);
			new (&m->get()->m_path) Path();
		}
		masked.get()->m_bone_masks.emplace(allocator);
	}
	~Controllers() { plain.get()->m_bone_masks.~Array(); masked.get()->m_bone_masks.~Array(); }
	RawStorage<anim::Controller> plain, masked;
};

// a stack of the scripted form: n instructions, kind[k] 1 = SAMPLE (slot, weight, time, looped), 2 = IK (alpha, target, leaf, bones)
void writeStack(OutputMemoryStream& bs, const uint32_t* kind, const uint32_t* slot, const float* weight, const uint32_t* time, const uint32_t* looped, uint32_t n) {
	bs.clear();
	for (uint32_t k = 0; k < n; ++k) {
		if (kind[k] == 1) {
			bs.write(anim::BlendStackInstructions::SAMPLE);
			bs.write(slot[k]);
			bs.write(weight[k]);
			bs.write(Time(time[k]));
			bs.write(looped[k] != 0);
		}
		else {
			bs.write(anim::BlendStackInstructions::IK);
			bs.write(0.0f); // alpha 0: evalIK returns before it looks the leaf bone up (controller.cpp:167), the model has no bone map here
			bs.write(Vec3(0.5f, 1.0f, 0.25f));
			bs.write(BoneNameHash());
			bs.write(u32(2));
		}
	}
	bs.write(anim::BlendStackInstructions::END);
}

// updateAnimator's :623-625 on one animator
void referenceStack(const anim::RuntimeContext& rc, Model* model, Pose* pose) {
	const uint32_t B = (uint32_t)model->m_bones.size();
	for (uint32_t k = 0; k < B; ++k) { // model->getRelativePose(*pose), model.cpp:226-237
		pose->positions[k] = model->m_bones[(int)k].relative_transform.pos;
		pose->rotations[k] = model->m_bones[(int)k].relative_transform.rot;
	}
	pose->is_absolute = false;
	anim::evalBlendStack(rc, *pose);
	pose->computeAbsolute(*model);
}

struct RenderSideAnimators {
	uint32_t* locks = nullptr;
	uint32_t* unlocks = nullptr;
	Pose* lockPose(EntityRef e) { ++locks[e.index]; return nullptr; }
	void unlockPose(EntityRef e, bool) { ++unlocks[e.index]; }
};

} // namespace

// One stack on one skeleton with clips[0 .. n_clips) in slots 0 .. n_clips (null slots where null_slot[s]): the absolute pose.
SHIM_API int ref_pose_stack(const RefSkeleton* sk, const RefClip* clips, uint32_t n_clips, const uint32_t* slot, const float* weight, const uint32_t* time,
	const uint32_t* looped, uint32_t n, float* pos, float* rot)
{
	IAllocator& allocator = getGlobalAllocator();
	RawStorage<Model> model_mem;
	Array<float> inv(allocator);
	buildModel(model_mem.get(), sk, inv, allocator);
	Array<RawStorage<Animation>*> anim_mem(allocator);
	Controllers controllers(allocator);
	{
		anim::RuntimeContext rc(*controllers.plain.get(), allocator);
		for (uint32_t c = 0; c < n_clips; ++c) {
			auto* m = new RawStorage<Animation>;
			anim_mem.push(m);
			buildAnimation(m->get(), clips[c], allocator);
			rc.animations.push(m->get());
		}
		rc.model = model_mem.get();
		Array<uint32_t> kind(allocator);
		for (uint32_t k = 0; k < n; ++k) kind.push(1);
		writeStack(rc.blendstack, kind.begin(), slot, weight, time, looped, n);
		Pose pose(allocator);
		pose.resize((int)sk->bone_count);
		referenceStack(rc, model_mem.get(), &pose);
		for (uint32_t b = 0; b < sk->bone_count; ++b) {
			pos[3 * b] = pose.positions[b].x; pos[3 * b + 1] = pose.positions[b].y; pos[3 * b + 2] = pose.positions[b].z;
			rot[4 * b] = pose.rotations[b].x; rot[4 * b + 1] = pose.rotations[b].y; rot[4 * b + 2] = pose.rotations[b].z; rot[4 * b + 3] = pose.rotations[b].w;
		}
	}
	for (RawStorage<Animation>* m : anim_mem) { destroyAnimation(m->get()); delete m; }
	destroyModel(model_mem.get());
	return 0;
}

// n_anim animators over n_models models (animator i: model model_of[i], controller masked when masked[i]).  Model m plays clips
// [clip_start[m], clip_start[m + 1]) in its slots 0 .. ; slot null_slot[m] (if < its clip count) is left null.  Frame f, animator i runs
// the stack of n_instr[f * n_anim + i] instructions at instr_start[f * n_anim + i] of the kind / slot / weight / time / looped columns.
// Outputs: the absolute poses of both sides after every frame, packed frame after frame and animator after animator; per frame and
// animator on_ref = 1 when side B left it to the reference path; info = {locks, unlocks: max and min over animators and frames of side
// B's counts per frame, rc}.
SHIM_API int ashim_run_animators(const RefSkeleton* sks, uint32_t n_models, const RefClip* clips, const uint32_t* clip_start, const uint32_t* null_slot,
	const uint32_t* model_of, const uint32_t* masked, uint32_t n_anim, uint32_t n_frames, const uint32_t* instr_start, const uint32_t* n_instr,
	const uint32_t* kind, const uint32_t* slot, const float* weight, const uint32_t* time, const uint32_t* looped,
	float* pos_ref, float* rot_ref, float* pos_b200, float* rot_b200, uint32_t* on_ref, uint32_t* info)
{
	lb200_ctx* ctx = nullptr;
	if (lb200_init(0, &ctx) != LB200_OK) return -1;
	IAllocator& allocator = getGlobalAllocator();
	int rc = 0;
	{
		Array<RawStorage<Model>*> model_mem(allocator);
		Array<Array<float>*> invs(allocator);
		for (uint32_t m = 0; m < n_models; ++m) {
			model_mem.push(new RawStorage<Model>);
			invs.push(new Array<float>(allocator));
			buildModel(model_mem[(int)m]->get(), &sks[m], *invs[(int)m], allocator);
		}
		Array<RawStorage<Animation>*> anim_mem(allocator);
		for (uint32_t c = 0; c < clip_start[n_models]; ++c) {
			anim_mem.push(new RawStorage<Animation>);
			buildAnimation(anim_mem[(int)c]->get(), clips[c], allocator);
		}
		Controllers controllers(allocator);
		Array<anim::RuntimeContext*> ctxs(allocator);
		Array<Pose*> poses_a(allocator), poses_b(allocator);
		Array<AnimatorB200Entry> entries(allocator);
		Array<uint32_t> locks(allocator), unlocks(allocator);
		locks.resize(n_anim);
		unlocks.resize(n_anim);
		for (uint32_t i = 0; i < n_anim; ++i) {
			const uint32_t m = model_of[i];
			auto* r = new anim::RuntimeContext(*(masked[i] ? controllers.masked.get() : controllers.plain.get()), allocator);
			for (uint32_t c = clip_start[m]; c < clip_start[m + 1]; ++c) r->animations.push(c - clip_start[m] == null_slot[m] ? nullptr : anim_mem[(int)c]->get());
			r->model = model_mem[(int)m]->get();
			ctxs.push(r);
			Pose* pa = new Pose(allocator); pa->resize((int)sks[m].bone_count); poses_a.push(pa);
			Pose* pb = new Pose(allocator); pb->resize((int)sks[m].bone_count); poses_b.push(pb);
		}
		RenderSideAnimators render;
		render.locks = locks.begin();
		render.unlocks = unlocks.begin();
		uint32_t max_lu = 0, min_lu = 0xffffffffu;
		size_t off = 0;
		{
			AnimatorsB200<RenderSideAnimators> b200(allocator);
			for (uint32_t f = 0; f < n_frames && rc == 0; ++f) {
				entries.clear();
				for (uint32_t i = 0; i < n_anim; ++i) {
					const uint32_t s = instr_start[f * n_anim + i];
					writeStack(ctxs[(int)i]->blendstack, kind + s, slot + s, weight + s, time + s, looped + s, n_instr[f * n_anim + i]);
					referenceStack(*ctxs[(int)i], model_mem[(int)model_of[i]]->get(), poses_a[(int)i]); // side A
					locks[i] = unlocks[i] = 0;
					render.lockPose(EntityRef{(i32)i}); // the graph part's lockPose (:614)
					entries.push({EntityRef{(i32)i}, model_mem[(int)model_of[i]]->get(), ctxs[(int)i], poses_b[(int)i]});
				}
				if (!b200.update(ctx, render, Span<const AnimatorB200Entry>(entries.begin(), entries.size()))) rc = -2;
				for (uint32_t i = 0; i < n_anim; ++i) on_ref[f * n_anim + i] = 0;
				for (u32 i : b200.referencePath()) { // the module's reference path for the animators left to it
					on_ref[f * n_anim + i] = 1;
					referenceStack(*ctxs[(int)i], model_mem[(int)model_of[i]]->get(), poses_b[(int)i]);
					render.unlockPose(EntityRef{(i32)i}, true);
				}
				for (uint32_t i = 0; i < n_anim; ++i) {
					max_lu = std::max(max_lu, std::max(locks[i], unlocks[i]));
					min_lu = std::min(min_lu, std::min(locks[i], unlocks[i]));
					const uint32_t B = sks[model_of[i]].bone_count;
					for (uint32_t k = 0; k < B; ++k) {
						const Pose& a = *poses_a[(int)i];
						const Pose& b = *poses_b[(int)i];
						float* pa = pos_ref + (off + k) * 3; float* ra = rot_ref + (off + k) * 4;
						float* pb = pos_b200 + (off + k) * 3; float* rb = rot_b200 + (off + k) * 4;
						pa[0] = a.positions[k].x; pa[1] = a.positions[k].y; pa[2] = a.positions[k].z;
						ra[0] = a.rotations[k].x; ra[1] = a.rotations[k].y; ra[2] = a.rotations[k].z; ra[3] = a.rotations[k].w;
						pb[0] = b.positions[k].x; pb[1] = b.positions[k].y; pb[2] = b.positions[k].z;
						rb[0] = b.rotations[k].x; rb[1] = b.rotations[k].y; rb[2] = b.rotations[k].z; rb[3] = b.rotations[k].w;
					}
					off += B;
				}
			}
		}
		info[0] = max_lu; info[1] = min_lu; info[2] = (uint32_t)rc;
		for (uint32_t i = 0; i < n_anim; ++i) { delete ctxs[(int)i]; delete poses_a[(int)i]; delete poses_b[(int)i]; }
		for (RawStorage<Animation>* m : anim_mem) { destroyAnimation(m->get()); delete m; }
		for (uint32_t m = 0; m < n_models; ++m) { destroyModel(model_mem[(int)m]->get()); delete invs[(int)m]; delete model_mem[(int)m]; }
	}
	lb200_shutdown(ctx);
	return rc;
}
