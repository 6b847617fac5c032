// TEST INFRASTRUCTURE — not product code.  The animator harness (ref_animators_harness.cpp, included whole: its Model / Animation /
// Controller stand-ins and its updateAnimator reference path) with IK instructions, over Models that have a bone map (bone i named
// BoneNameHash::fromU64(IK_BONE_HASH + i)), so that the reference's own evalIK finds its leaf.  Built (through
// ref_root_motion_harness.cpp) into oracle/_ref/libanimation_shim_b200.so by oracle/build_ref.py.
//   ref_pose_stack_ik:      Model::getRelativePose + evalBlendStack + Pose::computeAbsolute on one scripted stack of SAMPLE and IK
//                           instructions (tests/golden/ik_kat.npz)
//   ashim_run_animators_ik: ashim_run_animators with IK instructions and ctx.weight per animator (tests/test_animation_animators_ik_gpu.py)
//   ref_ik_math:            the reference's own vec3ToVec3, nlerp, LocalRigidTransform::inverted, length, conjugated on arrays
#include "ref_animators_harness.cpp"

namespace {

// IK instructions of the scripted form, one entry per instruction (read where kind is 2): leaf = bone index (named IK_BONE_HASH + leaf;
// an index the model does not have names a bone its map lacks), bone count, alpha, target xyz
struct IkColumns { const uint32_t* leaf; const uint32_t* bones; const float* alpha; const float* target3; };
constexpr u64 IK_BONE_HASH = 0x1b00000000ull;

void writeStackIk(OutputMemoryStream& bs, const uint32_t* kind, const uint32_t* slot, const float* weight, const uint32_t* time, const uint32_t* looped,
	const IkColumns& ik, uint32_t n)
{
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
			bs.write(ik.alpha[k]);
			bs.write(Vec3(ik.target3[3 * k], ik.target3[3 * k + 1], ik.target3[3 * k + 2]));
			bs.write(StableHash::fromU64(IK_BONE_HASH + ik.leaf[k]));
			bs.write(ik.bones[k]);
		}
	}
	bs.write(anim::BlendStackInstructions::END);
}

// buildModel plus the bone map Model::load fills (model.cpp:361): bone i is named IK_BONE_HASH + i
void buildModelWithBoneMap(Model* model, const RefSkeleton* sk, Array<float>& inv, IAllocator& allocator) {
	buildModel(model, sk, inv, allocator);
	new (&model->m_bone_map) Model::BoneMap(allocator);
	for (uint32_t i = 0; i < sk->bone_count; ++i) model->m_bone_map.insert(StableHash::fromU64(IK_BONE_HASH + i), (int)i);
}
void destroyModelWithBoneMap(Model* model) {
	using BoneMap = Model::BoneMap;
	model->m_bone_map.~BoneMap();
	destroyModel(model);
}

// ashim_run_animators over Models with bone maps, with the IK columns and ctx.weight ctx_weight[i] per animator (the loop of
// ashim_run_animators with those three differences)
int runAnimatorsIk(const RefSkeleton* sks, uint32_t n_models, const RefClip* clips, const uint32_t* clip_start, const uint32_t* null_slot,
	const uint32_t* model_of, const uint32_t* masked, uint32_t n_anim, uint32_t n_frames, const uint32_t* instr_start, const uint32_t* n_instr,
	const uint32_t* kind, const uint32_t* slot, const float* weight, const uint32_t* time, const uint32_t* looped, const IkColumns& ik, const float* ctx_weight,
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
			buildModelWithBoneMap(model_mem[(int)m]->get(), &sks[m], *invs[(int)m], allocator);
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
			r->weight = ctx_weight[i];
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
		for (uint32_t m = 0; m < n_models; ++m) {
			destroyModelWithBoneMap(model_mem[(int)m]->get());
			delete invs[(int)m];
			delete model_mem[(int)m];
		}
	}
	lb200_shutdown(ctx);
	return rc;
}
} // namespace

// ashim_run_animators over Models with bone maps, with IK instructions (kind 2) read from the ik_* columns (IkColumns) and ctx.weight
// ctx_weight[i] for animator i (the factor evalBlendStack gives evalIK's alpha, controller.cpp:280)
SHIM_API int ashim_run_animators_ik(const RefSkeleton* sks, uint32_t n_models, const RefClip* clips, const uint32_t* clip_start, const uint32_t* null_slot,
	const uint32_t* model_of, const uint32_t* masked, uint32_t n_anim, uint32_t n_frames, const uint32_t* instr_start, const uint32_t* n_instr,
	const uint32_t* kind, const uint32_t* slot, const float* weight, const uint32_t* time, const uint32_t* looped,
	const uint32_t* ik_leaf, const uint32_t* ik_bones, const float* ik_alpha, const float* ik_target3, const float* ctx_weight,
	float* pos_ref, float* rot_ref, float* pos_b200, float* rot_b200, uint32_t* on_ref, uint32_t* info)
{
	return runAnimatorsIk(sks, n_models, clips, clip_start, null_slot, model_of, masked, n_anim, n_frames, instr_start, n_instr, kind, slot, weight, time,
		looped, IkColumns{ik_leaf, ik_bones, ik_alpha, ik_target3}, ctx_weight, pos_ref, rot_ref, pos_b200, rot_b200, on_ref, info);
}

// One stack of SAMPLE and IK instructions (kind 1 / 2, IkColumns) through the reference's own evalBlendStack on a Model with a bone map:
// the absolute pose.  ctx.weight is 1.
SHIM_API int ref_pose_stack_ik(const RefSkeleton* sk, const RefClip* clips, uint32_t n_clips, const uint32_t* kind, const uint32_t* slot, const float* weight,
	const uint32_t* time, const uint32_t* looped, const uint32_t* ik_leaf, const uint32_t* ik_bones, const float* ik_alpha, const float* ik_target3, uint32_t n,
	float* pos, float* rot)
{
	IAllocator& allocator = getGlobalAllocator();
	RawStorage<Model> model_mem;
	Array<float> inv(allocator);
	buildModelWithBoneMap(model_mem.get(), sk, inv, allocator);
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
		writeStackIk(rc.blendstack, kind, slot, weight, time, looped, IkColumns{ik_leaf, ik_bones, ik_alpha, ik_target3}, n);
		Pose pose(allocator);
		pose.resize((int)sk->bone_count);
		referenceStack(rc, model_mem.get(), &pose);
		for (uint32_t b = 0; b < sk->bone_count; ++b) {
			pos[3 * b] = pose.positions[b].x; pos[3 * b + 1] = pose.positions[b].y; pos[3 * b + 2] = pose.positions[b].z;
			rot[4 * b] = pose.rotations[b].x; rot[4 * b + 1] = pose.rotations[b].y; rot[4 * b + 2] = pose.rotations[b].z; rot[4 * b + 3] = pose.rotations[b].w;
		}
	}
	for (RawStorage<Animation>* m : anim_mem) { destroyAnimation(m->get()); delete m; }
	destroyModelWithBoneMap(model_mem.get());
	return 0;
}

// The reference's math on n inputs: out_v2v[4] = Quat::vec3ToVec3(v0, v1), out_nlerp[4] = nlerp(qa, qb, t), out_inv[7] =
// LocalRigidTransform{lrt pos, lrt rot}.inverted(), out_len = length(v0), out_conj[4] = qa.conjugated()
SHIM_API int ref_ik_math(uint32_t n, const float* v0, const float* v1, const float* qa, const float* qb, const float* t, const float* lrt7,
	float* out_v2v, float* out_nlerp, float* out_inv, float* out_len, float* out_conj)
{
	for (uint32_t i = 0; i < n; ++i) {
		const Vec3 a(v0[3 * i], v0[3 * i + 1], v0[3 * i + 2]), b(v1[3 * i], v1[3 * i + 1], v1[3 * i + 2]);
		const Quat q = Quat::vec3ToVec3(a, b);
		out_v2v[4 * i] = q.x; out_v2v[4 * i + 1] = q.y; out_v2v[4 * i + 2] = q.z; out_v2v[4 * i + 3] = q.w;
		const Quat q1(qa[4 * i], qa[4 * i + 1], qa[4 * i + 2], qa[4 * i + 3]), q2(qb[4 * i], qb[4 * i + 1], qb[4 * i + 2], qb[4 * i + 3]);
		const Quat nl = nlerp(q1, q2, t[i]);
		out_nlerp[4 * i] = nl.x; out_nlerp[4 * i + 1] = nl.y; out_nlerp[4 * i + 2] = nl.z; out_nlerp[4 * i + 3] = nl.w;
		const float* l = lrt7 + 7 * i;
		const LocalRigidTransform inv = LocalRigidTransform{Vec3(l[0], l[1], l[2]), Quat(l[3], l[4], l[5], l[6])}.inverted();
		float* o = out_inv + 7 * i;
		o[0] = inv.pos.x; o[1] = inv.pos.y; o[2] = inv.pos.z; o[3] = inv.rot.x; o[4] = inv.rot.y; o[5] = inv.rot.z; o[6] = inv.rot.w;
		out_len[i] = length(a);
		const Quat c = q1.conjugated();
		out_conj[4 * i] = c.x; out_conj[4 * i + 1] = c.y; out_conj[4 * i + 2] = c.z; out_conj[4 * i + 3] = c.w;
	}
	return 0;
}
