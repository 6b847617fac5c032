// TEST INFRASTRUCTURE — not product code.  Runs the animation binding (lumixengine_b200/host/animation_b200.inl, compiled against the
// reference's own headers with the accessors of animation_b200_decl.inl patched into a temporary copy of animation.h by oracle/build_ref.py)
// over REAL Lumix::Model / Lumix::Animation / Lumix::Pose objects and next to the reference's own per-animable path:
//   side A: the body of AnimationModuleImpl::updateAnimable (animation_module.cpp:439-472) per animable — Model::getRelativePose,
//           Animation::getRelativePose (the reference's animation.cpp), Pose::computeAbsolute (the reference's pose.cpp), the time step
//   side B: AnimablesB200<RenderSide>::update — grouping by model, one lb200_animation per group on the GPU, poses written back through
//           lockPose / unlockPose, Animable::time advanced
// RenderSide is a three-function stand-in for RenderModule (getModelInstanceModel / lockPose / unlockPose, render_module.h:402-403): the
// engine's RenderModule has ~200 pure virtuals and needs the whole renderer; tests/test_integration_compile.py instantiates the same
// template with the real RenderModule type.  Model and Animation are engine Resources that cannot be constructed without the engine, so —
// like ref_anim_harness.cpp — their storage is zero-filled and the members the path reads are set by hand through `#define private public`.
#define private public
#define protected public
#include "animation/animation.h"
#include "renderer/model.h"
#include "renderer/pose.h"
#undef private
#undef protected
#include "animation/animation_module.h"
#include "core/default_allocator.h"
#include "core/log.h"
#include "engine/resource_manager.h"

#include <new>
#include <stdint.h>
#include <string.h>

#include "animation_b200.inl"

using namespace Lumix;

// link-time stand-ins for what resource.cpp / animation.cpp reference but this harness never reaches (as in ref_anim_harness.cpp)
namespace Lumix {
ResourceManagerHub::LoadHook::Action ResourceManagerHub::onBeforeLoad(Resource&) const { return LoadHook::Action::IMMEDIATE; }
Resource* ResourceManagerHub::load(ResourceType, const Path&) { return nullptr; }
const ResourceType Model::TYPE("model");
}

#define SHIM_API extern "C" __attribute__((visibility("default")))

namespace {

struct RefTrack { uint16_t bone_index, offset_bits; uint8_t bitsizes[3]; uint8_t skipped_channel; float min[3], to_range[3]; }; // = lb200_track
struct RefConstT { uint16_t bone_index, pad; float value[3]; };
struct RefConstR { uint16_t bone_index, pad; float value[4]; };
struct RefClip {
	float fps;
	uint32_t frame_count, t_bits, r_bits, n_t, n_ct, n_r, n_cr;
	const RefTrack* t; const RefConstT* ct; const RefTrack* r; const RefConstR* cr;
	const uint8_t* t_stream; uint32_t t_bytes; const uint8_t* r_stream; uint32_t r_bytes;
};
struct RefSkeleton { uint32_t bone_count; int32_t first_nonroot; const int16_t* parents; const float* bind_relative7; const float* inverse_bind7; };

template <typename T> struct RawStorage {
	RawStorage() { memset(mem, 0, sizeof(mem)); }
	T* get() { return reinterpret_cast<T*>(mem); }
	alignas(alignof(T)) unsigned char mem[sizeof(T)];
};

struct RenderSide { // what AnimationModuleImpl asks of RenderModule on this path
	Model* model = nullptr;
	Pose** poses = nullptr;
	uint32_t locks = 0, unlocks = 0;
	Model* getModelInstanceModel(EntityRef) { return model; }
	Pose* lockPose(EntityRef e) { ++locks; return poses[e.index]; }
	void unlockPose(EntityRef, bool) { ++unlocks; }
};

void buildAnimation(Animation* anim, const RefClip& clip, IAllocator& allocator) {
	new (&anim->m_translations) Array<Animation::TranslationTrack>(allocator);
	new (&anim->m_const_translations) Array<Animation::ConstTranslationTrack>(allocator);
	new (&anim->m_rotations) Array<Animation::RotationTrack>(allocator);
	new (&anim->m_const_rotations) Array<Animation::ConstRotationTrack>(allocator);
	new (&anim->m_mem) Array<u8>(allocator);
	for (uint32_t i = 0; i < clip.n_t; ++i) {
		Animation::TranslationTrack& t = anim->m_translations.emplace();
		t.bone_index = clip.t[i].bone_index;
		t.min = Vec3(clip.t[i].min[0], clip.t[i].min[1], clip.t[i].min[2]);
		t.to_range = Vec3(clip.t[i].to_range[0], clip.t[i].to_range[1], clip.t[i].to_range[2]);
		t.offset_bits = clip.t[i].offset_bits;
		memcpy(t.bitsizes, clip.t[i].bitsizes, 3);
	}
	for (uint32_t i = 0; i < clip.n_ct; ++i) {
		Animation::ConstTranslationTrack& t = anim->m_const_translations.emplace();
		t.bone_index = clip.ct[i].bone_index;
		t.value = Vec3(clip.ct[i].value[0], clip.ct[i].value[1], clip.ct[i].value[2]);
	}
	for (uint32_t i = 0; i < clip.n_r; ++i) {
		Animation::RotationTrack& t = anim->m_rotations.emplace();
		t.bone_index = clip.r[i].bone_index;
		t.min = Vec3(clip.r[i].min[0], clip.r[i].min[1], clip.r[i].min[2]);
		t.to_range = Vec3(clip.r[i].to_range[0], clip.r[i].to_range[1], clip.r[i].to_range[2]);
		t.offset_bits = clip.r[i].offset_bits;
		memcpy(t.bitsizes, clip.r[i].bitsizes, 3);
		t.skipped_channel = clip.r[i].skipped_channel;
	}
	for (uint32_t i = 0; i < clip.n_cr; ++i) {
		Animation::ConstRotationTrack& t = anim->m_const_rotations.emplace();
		t.bone_index = clip.cr[i].bone_index;
		t.value = Quat(clip.cr[i].value[0], clip.cr[i].value[1], clip.cr[i].value[2], clip.cr[i].value[3]);
	}
	// the file body as Animation::load keeps it (animation.cpp:437-440): both streams in m_mem, 8 bytes of padding behind them
	anim->m_mem.resize((int)(clip.t_bytes + clip.r_bytes + 8));
	memset(&anim->m_mem[0], 0, anim->m_mem.size());
	if (clip.t_bytes) memcpy(&anim->m_mem[0], clip.t_stream, clip.t_bytes);
	if (clip.r_bytes) memcpy(&anim->m_mem[clip.t_bytes], clip.r_stream, clip.r_bytes);
	anim->m_translation_stream = &anim->m_mem[0];
	anim->m_rotation_stream = &anim->m_mem[clip.t_bytes];
	anim->m_translations_frame_size_bits = clip.t_bits;
	anim->m_rotations_frame_size_bits = clip.r_bits;
	anim->m_frame_count = clip.frame_count;
	anim->m_fps = clip.fps;
	anim->m_max_accessed_bone_index = 0;
	anim->m_root_motion.rotation_track_idx = -1;
	anim->m_root_motion.translation_track_idx = -1;
	anim->m_current_state = Resource::State::READY;
}

void destroyAnimation(Animation* anim) {
	anim->m_translations.~Array();
	anim->m_const_translations.~Array();
	anim->m_rotations.~Array();
	anim->m_const_rotations.~Array();
	anim->m_mem.~Array();
}

} // namespace

// n_inst animables of one model: clip_index / time_ticks per animable (Animable::animation / ::time).  Outputs per side: absolute poses
// (n_inst x bone_count x 3 / x 4 floats), the advanced times, and info[0..3] = {locks, unlocks of side B, rc of side B, poses marked absolute}.
SHIM_API int ashim_run(const RefSkeleton* sk, const RefClip* clips, uint32_t n_clips, const uint32_t* clip_index, const uint32_t* time_ticks, uint32_t n_inst, float time_delta, uint32_t rounds,
	float* pos_ref, float* rot_ref, uint32_t* time_ref, float* pos_b200, float* rot_b200, uint32_t* time_b200, uint32_t* info)
{
	lb200_ctx* ctx = nullptr;
	if (lb200_init(0, &ctx) != LB200_OK) return -1;
	static DefaultAllocator allocator;
	const uint32_t B = sk->bone_count;
	int rc = 0;
	{
		RawStorage<Model> model_mem;
		Model* model = model_mem.get();
		new (&model->m_parents) Array<i16>(allocator);
		new (&model->m_bones) Array<Model::Bone>(allocator);
		Array<float> inv(allocator);
		inv.resize((int)B * 7);
		for (uint32_t i = 0; i < B; ++i) {
			model->m_parents.push(sk->parents[i]);
			Model::Bone& b = model->m_bones.emplace(allocator);
			const float* r = sk->bind_relative7 + 7 * i;
			b.relative_transform.pos = Vec3(r[0], r[1], r[2]);
			b.relative_transform.rot = Quat(r[3], r[4], r[5], r[6]);
			for (int c = 0; c < 7; ++c) inv[(int)(c * B + i)] = sk->inverse_bind7[7 * i + c]; // SoA, model.h:70-78
		}
		model->m_inverse_bind.px = &inv[0]; model->m_inverse_bind.py = &inv[(int)B]; model->m_inverse_bind.pz = &inv[(int)(2 * B)];
		model->m_inverse_bind.rx = &inv[(int)(3 * B)]; model->m_inverse_bind.ry = &inv[(int)(4 * B)]; model->m_inverse_bind.rz = &inv[(int)(5 * B)]; model->m_inverse_bind.rw = &inv[(int)(6 * B)];
		model->m_first_nonroot_bone_index = sk->first_nonroot;
		model->m_current_state = Resource::State::READY;

		Array<RawStorage<Animation>*> anim_mem(allocator);
		for (uint32_t c = 0; c < n_clips; ++c) {
			auto* m = new RawStorage<Animation>;
			anim_mem.push(m);
			buildAnimation(m->get(), clips[c], allocator);
		}
		Array<Animable> side_a(allocator), side_b(allocator);
		Array<Pose*> poses_a(allocator), poses_b(allocator);
		for (uint32_t i = 0; i < n_inst; ++i) {
			Animable a;
			a.time = Time(time_ticks[i]);
			a.animation = anim_mem[(int)clip_index[i]]->get();
			a.entity = EntityRef{(i32)i};
			side_a.push(a);
			side_b.push(a);
			Pose* pa = new Pose(allocator); pa->resize((int)B); poses_a.push(pa);
			Pose* pb = new Pose(allocator); pb->resize((int)B); poses_b.push(pb);
		}
		RenderSide render_b;
		render_b.model = model;
		render_b.poses = poses_b.begin();
		{
			AnimablesB200<RenderSide> b200(allocator);
			for (uint32_t round = 0; round < rounds && rc == 0; ++round) {
				// side A: AnimationModuleImpl::updateAnimable, animation_module.cpp:439-472, for every animable
				for (uint32_t i = 0; i < n_inst; ++i) {
					Animable& animable = side_a[(int)i];
					Pose* pose = poses_a[(int)i];
					for (uint32_t k = 0; k < B; ++k) { // model->getRelativePose(*pose), model.cpp:226-237 (model.cpp itself needs the whole renderer to link)
						pose->positions[k] = model->m_bones[(int)k].relative_transform.pos;
						pose->rotations[k] = model->m_bones[(int)k].relative_transform.rot;
					}
					pose->is_absolute = false;
					Animation::SampleContext sc;
					sc.pose = pose;
					sc.model = model;
					sc.time = animable.time;
					animable.animation->getRelativePose(sc);
					pose->computeAbsolute(*model);
					if (time_delta > 0) {
						Time t = animable.time + Time::fromSeconds(time_delta);
						const Time l = animable.animation->getLength();
						t = t % l;
						animable.time = t;
					}
					else {
						const Time l = animable.animation->getLength();
						Time dt = Time::fromSeconds(-time_delta) % l;
						Time t = animable.time + l - dt;
						t = t % l;
						animable.time = t;
					}
				}
				// side B
				if (!b200.update(ctx, render_b, Span<Animable>(side_b.begin(), side_b.size()), time_delta)) rc = -2;
			}
		}
		uint32_t absolute = 0;
		for (uint32_t i = 0; i < n_inst; ++i) {
			for (uint32_t k = 0; k < B; ++k) {
				const Pose& a = *poses_a[(int)i];
				const Pose& b = *poses_b[(int)i];
				float* pa = pos_ref + ((size_t)i * B + k) * 3; float* ra = rot_ref + ((size_t)i * B + k) * 4;
				float* pb = pos_b200 + ((size_t)i * B + k) * 3; float* rb = rot_b200 + ((size_t)i * B + k) * 4;
				pa[0] = a.positions[k].x; pa[1] = a.positions[k].y; pa[2] = a.positions[k].z;
				ra[0] = a.rotations[k].x; ra[1] = a.rotations[k].y; ra[2] = a.rotations[k].z; ra[3] = a.rotations[k].w;
				pb[0] = b.positions[k].x; pb[1] = b.positions[k].y; pb[2] = b.positions[k].z;
				rb[0] = b.rotations[k].x; rb[1] = b.rotations[k].y; rb[2] = b.rotations[k].z; rb[3] = b.rotations[k].w;
			}
			time_ref[i] = side_a[(int)i].time.raw();
			time_b200[i] = side_b[(int)i].time.raw();
			if (poses_b[(int)i]->is_absolute) ++absolute;
			delete poses_a[(int)i];
			delete poses_b[(int)i];
		}
		info[0] = render_b.locks; info[1] = render_b.unlocks; info[2] = (uint32_t)rc; info[3] = absolute;
		for (RawStorage<Animation>* m : anim_mem) { destroyAnimation(m->get()); delete m; }
		model->m_bones.~Array();
		model->m_parents.~Array();
	}
	lb200_shutdown(ctx);
	return rc;
}
