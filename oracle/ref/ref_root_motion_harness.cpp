// TEST INFRASTRUCTURE — not product code.  Animations with root motion: the IK animator harness (ref_animators_ik_harness.cpp, included
// whole: its Model / Animation stand-ins, bone maps, scripted stacks and reference paths) with Animation::m_root_motion constructed, every
// track named after its bone (BoneNameHash IK_BONE_HASH + bone index, the names of the bone map) and the reference's own
// Animation::setRootMotionBone run once on the freshly built clip.  Built into oracle/_ref/libanimation_shim_b200.so by
// oracle/build_ref.py, with the harnesses it includes in turn: one library for all of them.
//   ref_rm_tables:         setRootMotionBone's pose_translations / pose_rotations and track indices (tests/golden/root_motion_kat.npz)
//   ref_rm_pose_stack:     Model::getRelativePose + evalBlendStack + Pose::computeAbsolute on one stack of samples over such clips
//   ref_rm_math:           the reference's normalize(Quat) and Animation::getRotation on arrays
//   ashim_run_animables_rm / ashim_run_animators_rm: AnimablesB200 / AnimatorsB200 over such clips next to updateAnimable / evalBlendStack
//                          (tests/test_animation_root_motion_binding_gpu.py)
#include "ref_animators_ik_harness.cpp"

namespace {

// buildAnimation + m_flags, m_root_motion and the track names, then setRootMotionBone(name of root_bone) as Animation::onBeforeReady
// calls it (animation.cpp:392)
void buildAnimationRm(Animation* anim, const RefClip& clip, uint32_t flags, uint32_t root_bone, IAllocator& allocator) {
	buildAnimation(anim, clip, allocator);
	new (&anim->m_root_motion) Animation::RootMotion(allocator);
	for (Animation::TranslationTrack& t : anim->m_translations) t.bone_name = BoneNameHash::fromU64(IK_BONE_HASH + t.bone_index);
	for (Animation::ConstTranslationTrack& t : anim->m_const_translations) t.bone_name = BoneNameHash::fromU64(IK_BONE_HASH + t.bone_index);
	for (Animation::RotationTrack& t : anim->m_rotations) t.bone_name = BoneNameHash::fromU64(IK_BONE_HASH + t.bone_index);
	for (Animation::ConstRotationTrack& t : anim->m_const_rotations) t.bone_name = BoneNameHash::fromU64(IK_BONE_HASH + t.bone_index);
	anim->m_flags = (Animation::Flags)flags;
	anim->setRootMotionBone(BoneNameHash::fromU64(IK_BONE_HASH + root_bone));
}

void destroyAnimationRm(Animation* anim) {
	using RootMotion = Animation::RootMotion;
	anim->m_root_motion.~RootMotion();
	destroyAnimation(anim);
}

void writePose(const Pose& pose, uint32_t B, float* pos, float* rot) {
	for (uint32_t k = 0; k < B; ++k) {
		pos[3 * k] = pose.positions[k].x; pos[3 * k + 1] = pose.positions[k].y; pos[3 * k + 2] = pose.positions[k].z;
		rot[4 * k] = pose.rotations[k].x; rot[4 * k + 1] = pose.rotations[k].y; rot[4 * k + 2] = pose.rotations[k].z; rot[4 * k + 3] = pose.rotations[k].w;
	}
}

} // namespace

// setRootMotionBone on one clip: out3 = {translation_track_idx, rotation_track_idx, entries of pose_translations (0 when it returned
// early, else frame_count + 1)}; pose_t / pose_r receive that many entries.
SHIM_API int ref_rm_tables(const RefClip* clip, uint32_t flags, uint32_t root_bone, float* pose_t, float* pose_r, int32_t* out3) {
	IAllocator& allocator = getGlobalAllocator();
	RawStorage<Animation> mem;
	Animation* a = mem.get();
	buildAnimationRm(a, *clip, flags, root_bone, allocator);
	out3[0] = a->m_root_motion.translation_track_idx;
	out3[1] = a->m_root_motion.rotation_track_idx;
	out3[2] = (int32_t)a->m_root_motion.pose_translations.size();
	for (int f = 0; f < (int)a->m_root_motion.pose_translations.size(); ++f) {
		const Vec3 p = a->m_root_motion.pose_translations[f];
		const Quat q = a->m_root_motion.pose_rotations[f];
		pose_t[3 * f] = p.x; pose_t[3 * f + 1] = p.y; pose_t[3 * f + 2] = p.z;
		pose_r[4 * f] = q.x; pose_r[4 * f + 1] = q.y; pose_r[4 * f + 2] = q.z; pose_r[4 * f + 3] = q.w;
	}
	destroyAnimationRm(a);
	return 0;
}

// One stack of n samples (slot, weight, time, looped) over clips[0 .. n_clips), clip c with m_flags flags[c] and root_bone's root motion.
SHIM_API int ref_rm_pose_stack(const RefSkeleton* sk, const RefClip* clips, const uint32_t* flags, uint32_t n_clips, uint32_t root_bone, const uint32_t* slot,
	const float* weight, const uint32_t* time, const uint32_t* looped, uint32_t n, float* pos, float* rot)
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
			buildAnimationRm(m->get(), clips[c], flags[c], root_bone, allocator);
			rc.animations.push(m->get());
		}
		rc.model = model_mem.get();
		Array<uint32_t> kind(allocator);
		for (uint32_t k = 0; k < n; ++k) kind.push(1);
		writeStack(rc.blendstack, kind.begin(), slot, weight, time, looped, n);
		Pose pose(allocator);
		pose.resize((int)sk->bone_count);
		referenceStack(rc, model_mem.get(), &pose);
		writePose(pose, sk->bone_count, pos, rot);
	}
	for (RawStorage<Animation>* m : anim_mem) { destroyAnimationRm(m->get()); delete m; }
	destroyModel(model_mem.get());
	return 0;
}

// out_norm[4] = normalize(q[4]) for n quaternions; out_rot[4] = Animation::getRotation(frames[i], rotation track `track`) of a clip
// without root motion for n_frames frames
SHIM_API int ref_rm_math(const float* q, uint32_t n, float* out_norm, const RefClip* clip, uint32_t track, const uint32_t* frames, uint32_t n_frames, float* out_rot) {
	for (uint32_t i = 0; i < n; ++i) {
		const Quat r = normalize(Quat(q[4 * i], q[4 * i + 1], q[4 * i + 2], q[4 * i + 3]));
		out_norm[4 * i] = r.x; out_norm[4 * i + 1] = r.y; out_norm[4 * i + 2] = r.z; out_norm[4 * i + 3] = r.w;
	}
	if (!clip || !n_frames) return 0;
	IAllocator& allocator = getGlobalAllocator();
	RawStorage<Animation> mem;
	Animation* a = mem.get();
	buildAnimation(a, *clip, allocator);
	for (uint32_t i = 0; i < n_frames; ++i) {
		const Quat r = a->getRotation(frames[i], a->m_rotations[(int)track]);
		out_rot[4 * i] = r.x; out_rot[4 * i + 1] = r.y; out_rot[4 * i + 2] = r.z; out_rot[4 * i + 3] = r.w;
	}
	destroyAnimation(a);
	return 0;
}

// ashim_run with root motion: n_inst animables of one model, clip c with m_flags flags[c] and root_bone's root motion.  Every round, side A
// runs updateAnimable (animation_module.cpp:439-472) for every animable and side B runs AnimablesB200::update.  Outputs per round: both
// sides' absolute poses (n_inst x bone_count x 3 / x 4 floats) and times; info = {locks, unlocks of side B over all rounds, rc}.
SHIM_API int ashim_run_animables_rm(const RefSkeleton* sk, const RefClip* clips, const uint32_t* flags, uint32_t n_clips, uint32_t root_bone,
	const uint32_t* clip_index, const uint32_t* time_ticks, uint32_t n_inst, float time_delta, uint32_t rounds,
	float* pos_ref, float* rot_ref, uint32_t* time_ref, float* pos_b200, float* rot_b200, uint32_t* time_b200, uint32_t* info)
{
	lb200_ctx* ctx = nullptr;
	if (lb200_init(0, &ctx) != LB200_OK) return -1;
	IAllocator& allocator = getGlobalAllocator();
	const uint32_t B = sk->bone_count;
	int rc = 0;
	{
		RawStorage<Model> model_mem;
		Model* model = model_mem.get();
		Array<float> inv(allocator);
		buildModel(model, sk, inv, allocator);
		Array<RawStorage<Animation>*> anim_mem(allocator);
		for (uint32_t c = 0; c < n_clips; ++c) {
			anim_mem.push(new RawStorage<Animation>);
			buildAnimationRm(anim_mem[(int)c]->get(), clips[c], flags[c], root_bone, allocator);
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
		// AnimationModuleImpl::updateAnimable, animation_module.cpp:439-472
		auto updateAnimable = [&](Animable& animable, Pose* pose) {
			for (uint32_t k = 0; k < B; ++k) { // model->getRelativePose(*pose), model.cpp:226-237
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
			const Time l = animable.animation->getLength();
			if (time_delta > 0) animable.time = (animable.time + Time::fromSeconds(time_delta)) % l;
			else animable.time = (animable.time + l - Time::fromSeconds(-time_delta) % l) % l;
		};
		RenderSide render_b;
		render_b.model = model;
		render_b.poses = poses_b.begin();
		{
			AnimablesB200<RenderSide> b200(allocator);
			for (uint32_t round = 0; round < rounds && rc == 0; ++round) {
				for (uint32_t i = 0; i < n_inst; ++i) updateAnimable(side_a[(int)i], poses_a[(int)i]);
				if (!b200.update(ctx, render_b, Span<Animable>(side_b.begin(), side_b.size()), time_delta)) rc = -2;
				for (uint32_t i = 0; i < n_inst; ++i) {
					const size_t o = (size_t)round * n_inst + i;
					writePose(*poses_a[(int)i], B, pos_ref + o * B * 3, rot_ref + o * B * 4);
					writePose(*poses_b[(int)i], B, pos_b200 + o * B * 3, rot_b200 + o * B * 4);
					time_ref[o] = side_a[(int)i].time.raw();
					time_b200[o] = side_b[(int)i].time.raw();
				}
			}
		}
		info[0] = render_b.locks; info[1] = render_b.unlocks; info[2] = (uint32_t)rc;
		for (uint32_t i = 0; i < n_inst; ++i) { delete poses_a[(int)i]; delete poses_b[(int)i]; }
		for (RawStorage<Animation>* m : anim_mem) { destroyAnimationRm(m->get()); delete m; }
		destroyModel(model);
	}
	lb200_shutdown(ctx);
	return rc;
}

// ashim_run_animators_ik with root motion: the clips of model m are clips[clip_start[m] .. clip_start[m + 1]), clip c with m_flags
// flags[c] and root_bone's root motion; everything else (columns, outputs) as ashim_run_animators_ik.
SHIM_API int ashim_run_animators_rm(const RefSkeleton* sks, uint32_t n_models, const RefClip* clips, const uint32_t* flags, uint32_t root_bone,
	const uint32_t* clip_start, const uint32_t* null_slot, const uint32_t* model_of, const uint32_t* masked, uint32_t n_anim, uint32_t n_frames,
	const uint32_t* instr_start, const uint32_t* n_instr, const uint32_t* kind, const uint32_t* slot, const float* weight, const uint32_t* time,
	const uint32_t* looped, const uint32_t* ik_leaf, const uint32_t* ik_bones, const float* ik_alpha, const float* ik_target3,
	float* pos_ref, float* rot_ref, float* pos_b200, float* rot_b200, uint32_t* on_ref, uint32_t* info)
{
	lb200_ctx* ctx = nullptr;
	if (lb200_init(0, &ctx) != LB200_OK) return -1;
	IAllocator& allocator = getGlobalAllocator();
	const IkColumns ik{ik_leaf, ik_bones, ik_alpha, ik_target3};
	int rc = 0;
	{
		Array<RawStorage<Model>*> model_mem(allocator);
		Array<Array<float>*> invs(allocator);
		for (uint32_t m = 0; m < n_models; ++m) {
			model_mem.push(new RawStorage<Model>);
			invs.push(new Array<float>(allocator));
			buildModelWithBoneMap(model_mem[(int)m]->get(), &sks[m], *invs[(int)m], allocator);
		}
		Array<RawStorage<Animation>*> anim_mem(allocator);
		for (uint32_t c = 0; c < clip_start[n_models]; ++c) {
			anim_mem.push(new RawStorage<Animation>);
			buildAnimationRm(anim_mem[(int)c]->get(), clips[c], flags[c], root_bone, allocator);
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
					writeStackIk(ctxs[(int)i]->blendstack, kind + s, slot + s, weight + s, time + s, looped + s,
						IkColumns{ik.leaf + s, ik.bones + s, ik.alpha + s, ik.target3 + 3 * (size_t)s}, n_instr[f * n_anim + i]);
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
					writePose(*poses_a[(int)i], B, pos_ref + off * 3, rot_ref + off * 4);
					writePose(*poses_b[(int)i], B, pos_b200 + off * 3, rot_b200 + off * 4);
					off += B;
				}
			}
		}
		info[0] = max_lu; info[1] = min_lu; info[2] = (uint32_t)rc;
		for (uint32_t i = 0; i < n_anim; ++i) { delete ctxs[(int)i]; delete poses_a[(int)i]; delete poses_b[(int)i]; }
		for (RawStorage<Animation>* m : anim_mem) { destroyAnimationRm(m->get()); delete m; }
		for (uint32_t m = 0; m < n_models; ++m) {
			destroyModelWithBoneMap(model_mem[(int)m]->get());
			delete invs[(int)m];
			delete model_mem[(int)m];
		}
	}
	lb200_shutdown(ctx);
	return rc;
}
