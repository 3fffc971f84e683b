/* ORACLE — test infrastructure only. C API of the CPU restatement of bepuphysics2's solver + integrator path.
 * Consumes exactly the buffers the reference holds (128-B AOS BodyDynamics, AOSOA-W type batches) and mutates them in
 * place, like Simulation.Solve (BepuPhysics/Simulation.cs:L278-290) does. Parity: constraint functions / wide math / pose integration pinned to the reference's C# text
 * (oracle/ref_transpile, tests/test_oracle_pinned_to_reference.py); the driver in bepu_oracle.cpp unpinned (see bepu_math.h).
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load this. */
#ifndef BEPU_ORACLE_H
#define BEPU_ORACLE_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct oracle_type_batch {
    int32_t type_id;
    int32_t constraint_count;     /* TypeBatch.ConstraintCount (includes interior holes in the fallback batch) */
    int32_t* body_references;     /* AOSOA: [bundle][body slot][W] */
    float* prestep;               /* AOSOA: [bundle][prestep row][W] */
    float* accumulated_impulses;  /* AOSOA: [bundle][dof row][W] */
} oracle_type_batch;

typedef struct oracle_batch {
    int32_t type_batch_count;
    oracle_type_batch* type_batches;
} oracle_batch;

/* Optional velocity terms applied after the declarative callback wherever its result is kept (bepucuda_set_body_accelerations /
 * bepucuda_set_point_gravity in include/bepucuda.h). All zero: no terms. */
typedef struct oracle_integrator_terms {
    const float* accelerations;   /* body_count x 8 floats {a.xyz 0 | alpha.xyz 0} (PerBodyGravityDemo), or NULL */
    int32_t point_gravity;        /* nonzero: PlanetDemo's attractor at center with strength */
    float center[3];
    float strength;
} oracle_integrator_terms;

typedef struct oracle_scene {
    float* bodies;                /* body_count x 32 floats (BepuPhysics/BodyProperties.cs:L11-46,L318-338) */
    int32_t body_count;
    int32_t batch_count;
    oracle_batch* batches;
    int32_t bundle_width;         /* Vector<float>.Count of the emulated host */
    int32_t substep_count;
    const int32_t* velocity_iterations;  /* per substep */
    int32_t fallback_batch_threshold;
    float gravity[3];
    float linear_damping;
    float angular_damping;
    int32_t angular_integration_mode;
    int32_t allow_substeps_for_unconstrained;
    int32_t integrate_velocity_for_kinematics;
    const int32_t* constrained_kinematics;  /* body indices */
    int32_t constrained_kinematic_count;
    int32_t threads;              /* OpenMP threads for synchronized batches (fallback batch is always sequential) */
    int32_t simd;                 /* 0: scalar-per-lane evaluation; 1: 8-wide vector evaluation (requires bundle_width == 8) */
    oracle_integrator_terms terms;
} oracle_scene;

/* PrepareConstraintIntegrationResponsibilities + Solver.Solve + PoseIntegrator.IntegrateAfterSubstepping. 0 on success. */
int32_t oracle_solve(oracle_scene* scene, float dt);
/* Registry query. Returns 0 if the type is known. */
int32_t oracle_type_info(int32_t type_id, int32_t* bodies, int32_t* prestep_floats, int32_t* impulse_floats);
/* Single bundle entry points for unit tests: evaluate WarmStart / Solve of `type_id` on `lanes` constraints laid out as
 * one AOSOA bundle of width `lanes`; body state given per slot as SoA-free arrays of 32-float AOS records. */
int32_t oracle_max_threads(void);
/* NarrowPhase.RedistributeImpulses (NarrowPhaseConstraintUpdate.cs:L81-135) and its application to a whole contact type batch (same-type update). */
void oracle_redistribute_impulses(int32_t old_count, const int32_t* old_ids, float* old_impulses, int32_t new_count, const int32_t* new_ids, float* new_impulses);
int32_t oracle_update_contact_impulses(int32_t type_id, int32_t constraint_count, int32_t bundle_width, float* accumulated_impulses, const int32_t* old_feature_ids,
                                       const int32_t* new_feature_ids);

/* Solver.Add's first-fit batch search (Solver.cs:L1182-1199) over a whole constraint list in ascending key order (keys as documented for
 * bepucuda_color_constraints in include/bepucuda.h). Returns the number of batches, negative on bad arguments. */
int32_t oracle_first_fit_batches(int32_t constraint_count, int32_t bodies_per_constraint, const int32_t* encoded_body_references, int32_t body_count,
                                 int32_t fallback_threshold, int32_t order, const uint32_t* priorities, int32_t* batch_indices_out);

#ifdef __cplusplus
}
#endif
#endif
