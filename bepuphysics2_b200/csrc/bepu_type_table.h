// The constraint types of libbepucuda, one row per BatchTypeId. The planner, its byte model (get_type_info) and the host mirror read them here;
// every build of the device structs checks its row counts against them (bepu_joints_more.cuh). Plain C++: no CUDA.
// Read / written: the floats of body state the type's Solve and WarmStart access filters move, summed over its bodies. Per body
// (IBodyAccessFilter.cs:L38-126): All 20 / 6, NoPosition 17 / 6, NoOrientation 16 / 6, NoPose 13 / 6, OnlyAngular 13 / 3,
// OnlyAngularWithoutPose 9 / 3, OnlyLinear 7 / 3. Each row cites the TypeProcessor declaration that names the filters, per body, WarmStart's
// then Solve's; contacts access NoPose throughout.
#pragma once
#include <cstdint>

namespace bepucuda {

struct TypeRow {
    int32_t id;
    const char* name;
    int32_t bodies, prestep_rows, impulse_rows;  // floats of PrestepData / AccumulatedImpulses
    int32_t contacts;                            // per manifold; 0 for joints
    int32_t solve_read, solve_written, warm_start_read, warm_start_written;
};

inline constexpr TypeRow kTypeTable[] = {
    {0, "Contact1OneBody", 1, 11, 4, 1, 13, 6, 13, 6},             // ContactConvexTypes.cs:L334
    {1, "Contact2OneBody", 1, 15, 5, 2, 13, 6, 13, 6},             // ContactConvexTypes.cs:L489
    {2, "Contact3OneBody", 1, 19, 6, 3, 13, 6, 13, 6},             // ContactConvexTypes.cs:L654
    {3, "Contact4OneBody", 1, 23, 7, 4, 13, 6, 13, 6},             // ContactConvexTypes.cs:L829
    {4, "Contact1", 2, 14, 4, 1, 26, 12, 26, 12},                  // ContactConvexTypes.cs:L985
    {5, "Contact2", 2, 18, 5, 2, 26, 12, 26, 12},                  // ContactConvexTypes.cs:L1153
    {6, "Contact3", 2, 22, 6, 3, 26, 12, 26, 12},                  // ContactConvexTypes.cs:L1331
    {7, "Contact4", 2, 26, 7, 4, 26, 12, 26, 12},                  // ContactConvexTypes.cs:L1519
    {8, "Contact2NonconvexOneBody", 1, 18, 6, 2, 13, 6, 13, 6},    // ContactNonconvexTypes.cs:L187
    {9, "Contact3NonconvexOneBody", 1, 25, 9, 3, 13, 6, 13, 6},    // ContactNonconvexTypes.cs:L380
    {10, "Contact4NonconvexOneBody", 1, 32, 12, 4, 13, 6, 13, 6},  // ContactNonconvexTypes.cs:L578
    {15, "Contact2Nonconvex", 2, 21, 6, 2, 26, 12, 26, 12},        // ContactNonconvexTypes.cs:L104
    {16, "Contact3Nonconvex", 2, 28, 9, 3, 26, 12, 26, 12},        // ContactNonconvexTypes.cs:L295
    {17, "Contact4Nonconvex", 2, 35, 12, 4, 26, 12, 26, 12},       // ContactNonconvexTypes.cs:L491
    {22, "BallSocket", 2, 8, 3, 0, 40, 12, 34, 12},                // BallSocket.cs:L102
    {23, "AngularHinge", 2, 8, 2, 0, 26, 6, 22, 6},                // AngularHinge.cs:L225
    {24, "AngularSwivelHinge", 2, 8, 1, 0, 26, 6, 26, 6},          // AngularSwivelHinge.cs:L150
    {25, "SwingLimit", 2, 9, 1, 0, 26, 6, 26, 6},                  // SwingLimit.cs:L171
    {26, "TwistServo", 2, 14, 1, 0, 26, 6, 26, 6},                 // TwistServo.cs:L224
    {27, "TwistLimit", 2, 12, 1, 0, 26, 6, 26, 6},                 // TwistLimit.cs:L139
    {28, "TwistMotor", 2, 9, 1, 0, 26, 6, 26, 6},                  // TwistMotor.cs:L128
    {29, "AngularServo", 2, 9, 3, 0, 26, 6, 18, 6},                // AngularServo.cs:L140
    {30, "AngularMotor", 2, 5, 3, 0, 22, 6, 18, 6},                // AngularMotor.cs:L96
    {31, "Weld", 2, 9, 6, 0, 40, 12, 30, 12},                      // Weld.cs:L222
    {32, "VolumeConstraint", 4, 3, 1, 0, 28, 12, 28, 12},          // VolumeConstraint.cs:L188
    {33, "DistanceServo", 2, 12, 1, 0, 40, 12, 40, 12},            // DistanceServo.cs:L228
    {34, "DistanceLimit", 2, 10, 1, 0, 40, 12, 40, 12},            // DistanceLimit.cs:L183
    {35, "CenterDistanceConstraint", 2, 3, 1, 0, 14, 6, 14, 6},    // CenterDistanceConstraint.cs:L135
    {36, "AreaConstraint", 3, 3, 1, 0, 21, 9, 21, 9},              // AreaConstraint.cs:L199
    {37, "PointOnLineServo", 2, 14, 2, 0, 40, 12, 40, 12},         // PointOnLineServo.cs:L195
    {38, "LinearAxisServo", 2, 15, 1, 0, 40, 12, 40, 12},          // LinearAxisServo.cs:L250
    {39, "LinearAxisMotor", 2, 12, 1, 0, 40, 12, 40, 12},          // LinearAxisMotor.cs:L112
    {40, "LinearAxisLimit", 2, 13, 1, 0, 40, 12, 40, 12},          // LinearAxisLimit.cs:L153
    {41, "AngularAxisMotor", 2, 6, 1, 0, 26, 6, 22, 6},            // AngularAxisMotor.cs:L108
    {42, "OneBodyAngularServo", 1, 9, 3, 0, 13, 3, 13, 3},         // OneBodyAngularServo.cs:L111
    {43, "OneBodyAngularMotor", 1, 5, 3, 0, 13, 3, 9, 3},          // OneBodyAngularMotor.cs:L95
    {44, "OneBodyLinearServo", 1, 11, 3, 0, 20, 6, 20, 6},         // OneBodyLinearServo.cs:L148
    {45, "OneBodyLinearMotor", 1, 8, 3, 0, 17, 6, 17, 6},          // OneBodyLinearMotor.cs:L102
    {46, "SwivelHinge", 2, 14, 4, 0, 40, 12, 34, 12},              // SwivelHinge.cs:L216
    {47, "Hinge", 2, 14, 5, 0, 40, 12, 34, 12},                    // Hinge.cs:L224
    {52, "BallSocketMotor", 2, 8, 3, 0, 40, 12, 36, 12},           // BallSocketMotor.cs:L99
    {53, "BallSocketServo", 2, 11, 3, 0, 40, 12, 34, 12},          // BallSocketServo.cs:L109
    {54, "AngularAxisGearMotor", 2, 6, 1, 0, 22, 6, 22, 6},        // AngularAxisGearMotor.cs:L116
    {55, "CenterDistanceLimit", 2, 4, 1, 0, 14, 6, 14, 6},         // CenterDistanceLimit.cs:L134
};
inline constexpr int kTypeCount = sizeof(kTypeTable) / sizeof(TypeRow);

// The row of a type id; nullptr for an id without a type.
constexpr const TypeRow* type_row(int type_id) {
    for (const TypeRow& r : kTypeTable)
        if (r.id == type_id) return &r;
    return nullptr;
}

// Contacts per constraint of a type id; 0 for joints and ids without a type.
constexpr int32_t contact_count_of_type(int type_id) {
    const TypeRow* r = type_row(type_id);
    return r ? r->contacts : 0;
}

// The largest f(row) over the table: what a buffer sized for every type must hold.
template <class F>
constexpr int32_t max_over_types(F f) {
    int32_t m = 0;
    for (const TypeRow& r : kTypeTable) m = f(r) > m ? f(r) : m;
    return m;
}

}  // namespace bepucuda
