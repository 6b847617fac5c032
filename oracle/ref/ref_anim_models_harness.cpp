// TEST INFRASTRUCTURE — not product code.  The animation binding (lumixengine_b200/host/animation_b200.inl) over the animables of SEVERAL
// real Lumix::Models at once, next to the reference's own updateAnimable body per animable: AnimablesB200 keeps one group per model and
// poses all of them in one lb200_animation_update_many call.  Built (through ref_root_motion_harness.cpp) into
// oracle/_ref/libanimation_shim_b200.so by oracle/build_ref.py, against the same overlay of the reference and the same patched animation.h as ref_anim_shim_harness.cpp,
// whose stand-ins for Model / Animation construction (RawStorage, RefClip, buildAnimation ...) this file includes rather than repeats.
#include "ref_anim_shim_harness.cpp"

namespace {

// the members of a zero-filled Model the path reads: parents, bones' relative transforms, the SoA inverse bind pose (kept in `inv`)
void buildModel(Model* model, const RefSkeleton* sk, Array<float>& inv, IAllocator& allocator) {
	const uint32_t B = sk->bone_count;
	new (&model->m_parents) Array<i16>(allocator);
	new (&model->m_bones) Array<Model::Bone>(allocator);
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
}

void destroyModel(Model* model) {
	model->m_bones.~Array();
	model->m_parents.~Array();
}

// side A for one animable: the body of AnimationModuleImpl::updateAnimable, animation_module.cpp:439-472
void referenceUpdate(Animable& animable, Pose* pose, Model* model, float time_delta) {
	const uint32_t B = (uint32_t)model->m_bones.size();
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

// RenderModule stand-in for animables of several models: entity i is an instance of models[model_of[i]]
struct RenderSideModels {
	Model** models = nullptr;
	const uint32_t* model_of = nullptr;
	Pose** poses = nullptr;
	uint32_t locks = 0, unlocks = 0;
	Model* getModelInstanceModel(EntityRef e) { return models[model_of[e.index]]; }
	Pose* lockPose(EntityRef e) { ++locks; return poses[e.index]; }
	void unlockPose(EntityRef, bool) { ++unlocks; }
};

} // namespace

// ashim_run over the animables of several models (one AnimablesB200 group, one system of lb200_animation_update_many, per model):
// model m has skeleton sks[m] and clips [clip_start[m], clip_start[m + 1]) of `clips`; animable i plays clip clip_index[i] of model
// model_of[i] from time_ticks[i].  Poses are packed animable after animable, bone_count(model_of[i]) x 3 / x 4 floats each; info as
// ashim_run's.
SHIM_API int ashim_run_models(const RefSkeleton* sks, uint32_t n_models, const RefClip* clips, const uint32_t* clip_start, const uint32_t* model_of,
	const uint32_t* clip_index, const uint32_t* time_ticks, uint32_t n_inst, float time_delta, uint32_t rounds,
	float* pos_ref, float* rot_ref, uint32_t* time_ref, float* pos_b200, float* rot_b200, uint32_t* time_b200, uint32_t* info)
{
	lb200_ctx* ctx = nullptr;
	if (lb200_init(0, &ctx) != LB200_OK) return -1;
	static DefaultAllocator allocator;
	int rc = 0;
	{
		Array<RawStorage<Model>*> model_mem(allocator);
		Array<Array<float>*> invs(allocator);
		Array<Model*> models(allocator);
		for (uint32_t m = 0; m < n_models; ++m) {
			auto* mm = new RawStorage<Model>;
			auto* inv = new Array<float>(allocator);
			model_mem.push(mm);
			invs.push(inv);
			buildModel(mm->get(), &sks[m], *inv, allocator);
			models.push(mm->get());
		}
		Array<RawStorage<Animation>*> anim_mem(allocator);
		for (uint32_t c = 0; c < clip_start[n_models]; ++c) {
			auto* m = new RawStorage<Animation>;
			anim_mem.push(m);
			buildAnimation(m->get(), clips[c], allocator);
		}
		Array<Animable> side_a(allocator), side_b(allocator);
		Array<Pose*> poses_a(allocator), poses_b(allocator);
		for (uint32_t i = 0; i < n_inst; ++i) {
			const uint32_t m = model_of[i];
			Animable a;
			a.time = Time(time_ticks[i]);
			a.animation = anim_mem[(int)(clip_start[m] + clip_index[i])]->get();
			a.entity = EntityRef{(i32)i};
			side_a.push(a);
			side_b.push(a);
			Pose* pa = new Pose(allocator); pa->resize((int)sks[m].bone_count); poses_a.push(pa);
			Pose* pb = new Pose(allocator); pb->resize((int)sks[m].bone_count); poses_b.push(pb);
		}
		RenderSideModels render_b;
		render_b.models = models.begin();
		render_b.model_of = model_of;
		render_b.poses = poses_b.begin();
		{
			AnimablesB200<RenderSideModels> b200(allocator);
			for (uint32_t round = 0; round < rounds && rc == 0; ++round) {
				for (uint32_t i = 0; i < n_inst; ++i) referenceUpdate(side_a[(int)i], poses_a[(int)i], models[(int)model_of[i]], time_delta);
				if (!b200.update(ctx, render_b, Span<Animable>(side_b.begin(), side_b.size()), time_delta)) rc = -2;
			}
		}
		uint32_t absolute = 0;
		size_t off = 0; // bones of the animables before i
		for (uint32_t i = 0; i < n_inst; ++i) {
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
			time_ref[i] = side_a[(int)i].time.raw();
			time_b200[i] = side_b[(int)i].time.raw();
			if (poses_b[(int)i]->is_absolute) ++absolute;
			delete poses_a[(int)i];
			delete poses_b[(int)i];
		}
		info[0] = render_b.locks; info[1] = render_b.unlocks; info[2] = (uint32_t)rc; info[3] = absolute;
		for (RawStorage<Animation>* m : anim_mem) { destroyAnimation(m->get()); delete m; }
		for (uint32_t m = 0; m < n_models; ++m) { destroyModel(models[(int)m]); delete invs[(int)m]; delete model_mem[(int)m]; }
	}
	lb200_shutdown(ctx);
	return rc;
}
