//go:build !b200

package groth16

import (
	"github.com/consensys/gnark-crypto/ecc"
	"github.com/consensys/gnark/backend/accelerated/b200"
	"github.com/consensys/gnark/backend/groth16"
	"github.com/consensys/gnark/backend/witness"
	"github.com/consensys/gnark/constraint"
)

// Prove generates the proof of knowledge of a r1cs with full witness (secret + public part).
//
// NB! the provided proving key must be a B200 proving key. Initialize and deserialize the proving key using
// [NewProvingKey] and the serialization methods.
func Prove(r1cs constraint.ConstraintSystem, pk groth16.ProvingKey, fullWitness witness.Witness, opts ...b200.Option) (groth16.Proof, error) {
	panic("b200 backend requested but program compiled without 'b200' build tag")
}

// ProveBatch generates one proof per full witness of one r1cs in a single device call.
//
// NB! the provided proving key must be a B200 proving key.
func ProveBatch(r1cs constraint.ConstraintSystem, pk groth16.ProvingKey, fullWitnesses []witness.Witness, opts ...b200.Option) ([]groth16.Proof, error) {
	panic("b200 backend requested but program compiled without 'b200' build tag")
}

// Setup generates a proving and verifying key for a given r1cs.
//
// The method wraps the [groth16.Setup] method, but the returned proving key is a B200 proving key. To convert the key
// to a standard Groth16 proving key, use the serialization methods.
func Setup(r1cs constraint.ConstraintSystem) (groth16.ProvingKey, groth16.VerifyingKey, error) {
	panic("b200 backend requested but program compiled without 'b200' build tag")
}

// DummySetup generates a dummy proving key for a given circuit. It doesn't perform the precomputations and thus the
// returned proving key cannot be used to generate proofs. The method is useful for development and testing purposes.
func DummySetup(r1cs constraint.ConstraintSystem) (groth16.ProvingKey, error) {
	panic("b200 backend requested but program compiled without 'b200' build tag")
}

// NewProvingKey creates a new empty proving key for deserializing into.
//
// The method is compatible with [groth16.NewProvingKey], but returns a B200 proving key.
func NewProvingKey(curveID ecc.ID) groth16.ProvingKey {
	panic("b200 backend requested but program compiled without 'b200' build tag")
}
